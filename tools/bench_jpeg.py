"""Times the batched baseline-JPEG decoder (csrc/pv_jpeg.cu) on 256 frames of 340x256 4:2:0 at quality 90 - the frames
of 8 SlowFast clips of 32 - with CUDA events: decode_jpeg_frames end to end (host parse, one pinned staging copy,
three launches, the status read-back), each kernel on its own (torch.profiler kernel times over the same calls, in a
separate pass), and decode followed by clip_transform_batch to the 8 x 3 x 32 x 224^2 f16 model input.  When cv2 is
importable it also times cv2.imdecode + cvtColor over all the host's cores (a thread pool, cv2.setNumThreads(1) in
each worker), else it says the comparison was not run.  Reports frames/s and entropy-coded MB/s, and prints the card's
name, power limit and max SM clock first.  Frames are encoded with Pillow from seeded content (smooth gradients with
sensor-like noise).

The same frames are then encoded again with a restart marker after every MCU row (16 segments per frame instead of 1)
and the decode, kernel and cv2 times repeated: the entropy kernel runs one segment per CTA, so this shows what
spreading a batch over more SMs gives.

    python tools/bench_jpeg.py [--iters 20]
"""
import argparse
import io
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pytorchvideo_b200.data import decode_jpeg_frames, parse_jpeg  # noqa: E402
from pytorchvideo_b200.transforms import functional as Fv  # noqa: E402

N_CLIPS, T, H, W = 8, 32, 256, 340


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:              # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % e


def frames(n, seed=0, restart_rows=0):
    from PIL import Image
    r = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W].astype(np.float32)
    out = []
    for i in range(n):
        ph = i * 0.07
        img = np.stack([128 + 100 * np.sin(x / 23 + ph), 128 + 90 * np.cos(y / 17 - ph), 128 + 60 * np.sin((x + y) / 31)], -1)
        img = np.clip(img + r.normal(0, 8, img.shape), 0, 255).astype(np.uint8)
        bio = io.BytesIO()
        Image.fromarray(img).save(bio, "JPEG", quality=90, subsampling=2, restart_marker_rows=restart_rows)
        out.append(bio.getvalue())
    return out


def timed(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters        # ms


def entropy_bytes(blobs):
    total = 0
    for b in blobs:
        segs = parse_jpeg(b)[3]
        total += segs[-1][1] - segs[0][0]
    return total


def kernel_times(blobs, out, iters):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            decode_jpeg_frames(blobs, out=out)
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        if "jpeg_" in ev.key:
            name = ev.key.split("::")[-1].split("(")[0]
            kern[name] = getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0)) / iters / 1e3
    return kern


def time_decode(blobs, out, scan_bytes, iters):
    """decode_jpeg_frames end to end with CUDA events, then each kernel in a separate profiled pass"""
    n = len(blobs)
    segs = sum(parse_jpeg(b)[2].n_segments for b in blobs)
    ms = timed(lambda: decode_jpeg_frames(blobs, out=out), iters)
    print("decode_jpeg_frames (%d segments) %8.3f ms/batch  %9.0f frames/s  %7.1f entropy MB/s" % (
        segs, ms, n / ms * 1e3, scan_bytes / 1e6 / ms * 1e3))
    kern = kernel_times(blobs, out, iters)
    for name, t in sorted(kern.items()):
        extra = "  %7.1f entropy MB/s" % (scan_bytes / 1e6 / t * 1e3) if "huffman" in name else ""
        print("  kernel %-40s %8.3f ms/batch%s" % (name, t, extra))
    return {"segments": segs, "decode_ms": ms, "kernels_ms": kern}


def cpu_pool(blobs, iters, gpu_out):
    """cv2.imdecode + cvtColor over a pool of os.cpu_count() threads; None when cv2 is not importable"""
    try:
        import cv2
    except ImportError:
        print("cv2 not importable: the CPU thread-pool comparison was not run")
        return None
    cores = os.cpu_count() or 1
    arrs = [np.frombuffer(b, np.uint8) for b in blobs]

    def one(a):
        return cv2.cvtColor(cv2.imdecode(a, cv2.IMREAD_COLOR), cv2.COLOR_BGR2RGB)
    with ThreadPoolExecutor(max_workers=cores, initializer=lambda: cv2.setNumThreads(1)) as ex:
        ref = list(ex.map(one, arrs))
        t0 = time.perf_counter()
        for _ in range(iters):
            list(ex.map(one, arrs))
        ms = (time.perf_counter() - t0) * 1e3 / iters
    same = bool(np.array_equal(np.stack(ref), gpu_out.cpu().numpy()))
    print("cv2.imdecode pool (%d threads) %8.3f ms/batch  %9.0f frames/s  (GPU output bit-exact: %s)" % (
        cores, ms, len(blobs) / ms * 1e3, same))
    return {"threads": cores, "ms": ms, "bit_exact": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    print("card:", card())
    blobs = frames(N_CLIPS * T)
    n = len(blobs)
    scan_bytes = entropy_bytes(blobs)
    print("batch: %d frames %dx%d 4:2:0 q90, %.2f MB of files, %.2f MB entropy-coded, no restart markers" % (
        n, W, H, sum(len(b) for b in blobs) / 1e6, scan_bytes / 1e6))
    res = {"frames": n, "width": W, "height": H, "entropy_mb": scan_bytes / 1e6}
    out = torch.empty((n, H, W, 3), dtype=torch.uint8, device="cuda")
    res["no_restart"] = time_decode(blobs, out, scan_bytes, args.iters)

    # host-side part alone: parse of every stream (decode_jpeg_frames parses each frame once more, in place)
    t0 = time.perf_counter()
    for _ in range(args.iters):
        for b in blobs:
            parse_jpeg(b)
    host_ms = (time.perf_counter() - t0) * 1e3 / args.iters
    res["host_parse_ms"] = host_ms
    print("  host parse alone      %8.3f ms/batch (one thread)" % host_ms)

    mean, std = (0.45, 0.45, 0.45), (0.225, 0.225, 0.225)
    top, left = (H - 224) // 2, (W - 224) // 2

    def decode_transform():
        d = decode_jpeg_frames(blobs, out=out).view(N_CLIPS, T, H, W, 3).permute(0, 4, 1, 2, 3)
        return Fv.clip_transform_batch(d, window=(top, left, 224, 224), mean=mean, std=std, div255=True,
                                       out_dtype=torch.float16)
    y = decode_transform()
    assert tuple(y.shape) == (N_CLIPS, 3, T, 224, 224) and y.dtype == torch.float16
    ms2 = timed(decode_transform, args.iters)
    res["decode_transform_ms"] = ms2
    print("decode -> clip_transform_batch (8x3x32x224^2 f16) %8.3f ms/batch  %9.0f frames/s" % (ms2, n / ms2 * 1e3))
    res["no_restart"]["cpu"] = cpu_pool(blobs, args.iters, out)

    rblobs = frames(n, restart_rows=1)
    rscan = entropy_bytes(rblobs)
    print("same frames, a restart marker every MCU row: %.2f MB of files, %.2f MB entropy-coded" % (
        sum(len(b) for b in rblobs) / 1e6, rscan / 1e6))
    res["restart_every_row"] = time_decode(rblobs, out, rscan, args.iters)
    res["restart_every_row"]["cpu"] = cpu_pool(rblobs, args.iters, out)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
