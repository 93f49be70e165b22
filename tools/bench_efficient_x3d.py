"""Efficient X3D against X3D on the engine: ms per step and clips/s of efficient_x3d_xs / _s and x3d_xs / _s at one
batch size, with the x3d weights mapped onto the efficient tree (testing.map_x3d_to_efficient), so both run the same
network.  The pairs are timed alternately, several rounds each, with CUDA events around graph replays after a warm-up;
the card's name, power limit and SM clock are printed with the numbers.  Writes nothing.

    python tools/bench_efficient_x3d.py [--batch 32] [--steps 50] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pytorchvideo_b200 import testing as TS  # noqa: E402
from pytorchvideo_b200.models import hub as H  # noqa: E402


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def _time(m, x, steps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        m(x)
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to measure")
    print("card:", _card())
    results = {}
    for size, T in (("xs", 4), ("s", 13)):
        x3 = TS.randomize_model(getattr(H, "x3d_" + size)(), seed=5).eval()
        eff = TS.map_x3d_to_efficient(x3, getattr(H, "efficient_x3d_" + size)().eval())
        x = TS.synthetic_clip(a.batch, T, 160, 160, seed=8).cuda()
        models = {"x3d_" + size: x3.cuda(), "efficient_x3d_" + size: eff.cuda()}
        with torch.no_grad():
            outs = {k: m(x).clone() for k, m in models.items()}
            same = torch.equal(*outs.values())
            for m in models.values():
                for _ in range(a.warmup):
                    m(x)
            torch.cuda.synchronize()
            times = {k: [] for k in models}
            for _ in range(a.rounds):
                for k, m in models.items():
                    times[k].append(_time(m, x, a.steps))
        for k, ts in times.items():
            ts = sorted(ts)
            results[k] = {"batch": a.batch, "ms_per_step_median": ts[len(ts) // 2], "ms_per_step_min": ts[0],
                          "ms_per_step_max": ts[-1], "clips_per_s": a.batch * 1000.0 / ts[len(ts) // 2]}
        results["bitwise_equal_" + size] = same
        for m in models.values():
            m.cpu()
    print(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
