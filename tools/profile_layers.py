"""Per-layer timing of the SlowFast-R50 (batch 8) convolution shapes that dominate the bench step.

Each layer is built as a one-op plan, captured `--reps` times back to back in one CUDA graph and replayed; the time
per launch is the median over `--rounds` replays, timed with CUDA events.  Achieved GB/s and TFLOP/s use the
algorithmic bytes and FLOPs the plan records for the launch (Plan.meta), and `of bound` is the larger of
FLOPs / 989 TFLOP/s and bytes / 3.35 TB/s (H100 SXM data sheet, dense f16) over the measured time, with the binding
one named.  The card, its power limit and max SM clock are printed with the numbers.

  python tools/profile_layers.py [--reps 50] [--rounds 7] [--json out.json] [name-substring ...]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn as nn

from pytorchvideo_b200 import _lib as L
from pytorchvideo_b200 import testing as TS
from pytorchvideo_b200.engine.plan import Plan

PEAK_FLOPS = 989e12
PEAK_BYTES = 3.35e12

LAYERS = [
    # name, (N, Ci, T, H, W), Co, kernel, stride, padding, residual
    ("slow_stem_1x7x7_3to64", (8, 3, 8, 224, 224), 64, (1, 7, 7), (1, 2, 2), (0, 3, 3), False),
    ("fast_stem_5x7x7_3to8", (8, 3, 32, 224, 224), 8, (5, 7, 7), (1, 2, 2), (2, 3, 3), False),
    ("res2_conv_a_80to64", (8, 80, 8, 56, 56), 64, (1, 1, 1), (1, 1, 1), (0, 0, 0), False),
    ("res2_conv_a_256to64", (8, 256, 8, 56, 56), 64, (1, 1, 1), (1, 1, 1), (0, 0, 0), False),
    ("res2_conv_c_64to256_res", (8, 64, 8, 56, 56), 256, (1, 1, 1), (1, 1, 1), (0, 0, 0), True),
    ("res2_branch1_80to256", (8, 80, 8, 56, 56), 256, (1, 1, 1), (1, 1, 1), (0, 0, 0), False),
    ("res3_conv_a_512to128", (8, 512, 8, 28, 28), 128, (1, 1, 1), (1, 1, 1), (0, 0, 0), False),
    ("res3_conv_c_128to512_res", (8, 128, 8, 28, 28), 512, (1, 1, 1), (1, 1, 1), (0, 0, 0), True),
    ("res3_branch1_320to512_s2", (8, 320, 8, 56, 56), 512, (1, 1, 1), (1, 2, 2), (0, 0, 0), False),
    ("res4_conv_a_3x1x1_1024to256", (8, 1024, 8, 14, 14), 256, (3, 1, 1), (1, 1, 1), (1, 0, 0), False),
    ("res4_conv_c_256to1024_res", (8, 256, 8, 14, 14), 1024, (1, 1, 1), (1, 1, 1), (0, 0, 0), True),
    ("res4_branch1_640to1024_s2", (8, 640, 8, 28, 28), 1024, (1, 1, 1), (1, 2, 2), (0, 0, 0), False),
    ("res5_conv_a_3x1x1_2048to512", (8, 2048, 8, 7, 7), 512, (3, 1, 1), (1, 1, 1), (1, 0, 0), False),
    ("res5_conv_c_512to2048_res", (8, 512, 8, 7, 7), 2048, (1, 1, 1), (1, 1, 1), (0, 0, 0), True),
    ("res5_branch1_1280to2048_s2", (8, 1280, 8, 14, 14), 2048, (1, 1, 1), (1, 2, 2), (0, 0, 0), False),
    ("fast_res4_conv_c_32to128_res", (8, 32, 32, 14, 14), 128, (1, 1, 1), (1, 1, 1), (0, 0, 0), True),
]


def device_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit / max SM clock unavailable"
    return "%s, %d SMs, %s" % (name, torch.cuda.get_device_properties(0).multi_processor_count, q)


def build(dev, xs, co, k, s, p, use_res, name):
    g = torch.Generator().manual_seed(0)
    plan = Plan(dev, L.PV_F16)
    x = torch.randn(xs, generator=g).to(dev)
    xr = plan.emit_input_ncdhw(x, xs[1], 4 if xs[1] <= 4 else xs[1])
    w = torch.randn(co, xs[1], *k, generator=g) * (2.0 / (xs[1] * k[0] * k[1] * k[2])) ** 0.5
    bn = nn.BatchNorm3d(co).eval()
    To, Ho, Wo = [(xs[2 + i] + 2 * p[i] - k[i]) // s[i] + 1 for i in range(3)]
    rr = None
    if use_res:
        rr = plan.emit_input_ncdhw(torch.randn(xs[0], co, To, Ho, Wo, generator=g).to(dev), co, co)
    plan.emit_conv(xr, w, None, bn, s, p, (1, 1, 1), 1, L.ACT_RELU, rr, name)
    plan.finalize()
    return plan


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50, help="launches per CUDA graph")
    ap.add_argument("--rounds", type=int, default=7, help="graph replays; the median is reported")
    ap.add_argument("--json", default=None, help="also write the rows to this path")
    ap.add_argument("only", nargs="*", help="run only layers whose name contains one of these")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("profile_layers: no CUDA device")
    dev = torch.device("cuda:0")
    info = device_info()
    print(info, flush=True)
    print("%-30s %9s %8s %8s %6s %9s  %s" % ("layer", "us", "GB/s", "TFLOP/s", "bound", "of bound", "kernels"))
    rows = []
    for name, xs, co, k, s, p, use_res in LAYERS:
        if args.only and not any(o in name for o in args.only):
            continue
        plan = build(dev, xs, co, k, s, p, use_res, name)
        stream = torch.cuda.Stream(device=dev)
        with torch.cuda.stream(stream):
            plan.run(stream.cuda_stream, single_stream=True)     # layout conversions + one warm-up launch
        stream.synchronize()
        idx = [i for i, (n, _) in enumerate(plan.ops) if not n.startswith("ncdhw_to_ndhwc")]
        fns = [plan.ops[i][1] for i in idx]

        def layer_once():
            for fn in fns:
                fn(stream.cuda_stream)
            stream.synchronize()
        _, launched = TS.launched_kernels(layer_once)
        flops = sum(plan.meta[i]["flops"] for i in idx)
        nbytes = sum(plan.meta[i]["bytes"] for i in idx)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            sp = torch.cuda.current_stream().cuda_stream
            for _ in range(args.reps):
                for fn in fns:
                    fn(sp)
        with torch.cuda.stream(stream):
            graph.replay()                                       # warm-up replay
            times = []
            for _ in range(args.rounds):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                graph.replay()
                e1.record(stream)
                e1.synchronize()
                times.append(e0.elapsed_time(e1) * 1e3 / args.reps)
        us = statistics.median(times)
        t_tc, t_hbm = flops / PEAK_FLOPS, nbytes / PEAK_BYTES
        bound = "HBM" if t_hbm >= t_tc else "TC"
        share = max(t_tc, t_hbm) * 1e6 / us
        kernels = "+".join(sorted(launched))
        print("%-30s %9.1f %8.0f %8.1f %6s %8.0f%%  %s" % (name, us, nbytes / us / 1e3, flops / us / 1e6, bound,
                                                          100 * share, kernels), flush=True)
        rows.append({"layer": name, "us": us, "us_rounds": times, "bytes": nbytes, "flops": flops,
                     "bound": bound, "share_of_bound": share, "kernels": kernels})
        del graph
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"device": info, "reps": args.reps, "rounds": args.rounds, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
