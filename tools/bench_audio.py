"""Audio model timings on the GPU.

* AVSlowFast-R50 (create_audio_visual_slowfast, depth 50) at batch 8 next to slowfast_r50 on the same visual clips
  (slow 8x224^2, fast 32x224^2; AVSlowFast also gets a (8, 1, 128, 1, 80) spectrogram), the two alternated over
  ``--rounds`` rounds in one process; the median per model is reported.
* The acoustic ResNet-50 (create_acoustic_resnet) at batch 64 on (64, 1, 128, 1, 80).
* For scale: a separate in-place f16 broadcast add of fuse_a over the Slow concat tensor at the four fusion points
  (the pass the epilogue addend saves), timed as ATen ``add_`` on channels-last tensors of the same shapes.

Times are CUDA events over ``--iters`` CUDA-graph replays after ``--warmup``; the card's name, power limit and max SM
clock are read in the same run.

    python tools/bench_audio.py [--iters 20] [--warmup 5] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pytorchvideo_b200 import _lib as L, testing as TS  # noqa: E402
from pytorchvideo_b200 import models as M  # noqa: E402
from pytorchvideo_b200.engine import compile_model  # noqa: E402


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    L.require_device()
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"device": torch.cuda.get_device_name(0), "nvidia_smi": smi}), flush=True)

    import pytorchvideo_b200.models.hub as H
    B = 8
    visual = [t.to(dev) for t in TS.slowfast_inputs(torch.rand(B, 3, 32, 224, 224))]
    audio = torch.rand(B, 1, 128, 1, 80, device=dev)
    sf = TS.randomize_model(H.slowfast_r50(), seed=1234).eval().to(dev)
    av = TS.randomize_model(M.create_audio_visual_slowfast(), seed=1234).eval().to(dev)
    cm_sf = compile_model(sf, visual, dtype="f16")
    cm_av = compile_model(av, visual + [audio], dtype="f16")
    cm_sf(visual)
    cm_av(visual + [audio])
    t_sf, t_av = [], []
    for _ in range(a.rounds):
        t_sf.append(timed(cm_sf.graph.replay, a.iters, a.warmup))
        t_av.append(timed(cm_av.graph.replay, a.iters, a.warmup))
    print(json.dumps({"batch": B, "slowfast_r50_ms": round(statistics.median(t_sf), 3),
                      "avslowfast_r50_ms": round(statistics.median(t_av), 3),
                      "slowfast_r50_ms_all": [round(t, 3) for t in t_sf],
                      "avslowfast_r50_ms_all": [round(t, 3) for t in t_av],
                      "launches": {"slowfast_r50": cm_sf.plan.num_launches(),
                                   "avslowfast_r50": cm_av.plan.num_launches()}}), flush=True)
    del cm_sf, cm_av, sf
    torch.cuda.empty_cache()

    # the separate add pass the epilogue addend replaces: fuse_a (B, C, T, 1, 1) + the Slow concat (B, C, T, H, W)
    t_add = []
    for c, hw in ((80, 56), (320, 56), (640, 28), (1280, 14)):
        y = torch.zeros(B, c, 8, hw, hw, dtype=torch.float16, device=dev).to(memory_format=torch.channels_last_3d)
        fa = torch.rand(B, c, 8, 1, 1, dtype=torch.float16, device=dev)
        t_add.append(timed(lambda: y.add_(fa), a.iters, a.warmup))
    print(json.dumps({"separate_add_pass_ms": round(sum(t_add), 4), "per_fusion_point_ms": [round(t, 4) for t in t_add],
                      "bytes_moved_mb": round(sum(2 * 2 * B * c * 8 * hw * hw for c, hw in
                                                  ((80, 56), (320, 56), (640, 28), (1280, 14))) / 1e6, 1)}), flush=True)

    B = 64
    ac = TS.randomize_model(M.create_acoustic_resnet(), seed=1234).eval().to(dev)
    spec = torch.rand(B, 1, 128, 1, 80, device=dev)
    cm = compile_model(ac, spec, dtype="f16")
    cm(spec)
    t = [timed(cm.graph.replay, a.iters, a.warmup) for _ in range(a.rounds)]
    print(json.dumps({"batch": B, "acoustic_resnet50_ms": round(statistics.median(t), 3),
                      "acoustic_resnet50_ms_all": [round(v, 3) for v in t]}), flush=True)


if __name__ == "__main__":
    main()
