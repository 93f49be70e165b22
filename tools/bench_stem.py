"""Temporal stems on the H100: the streaming kernel and the factored route, per shape.

    python tools/bench_stem.py [--launches 50] [--rounds 7] [--out DIR]

Each route of one stem shape is built in one process (the SM count the planner routes by, plan.H100_SXM_SMS, is patched
per plan build: down to 1, so the stream route is also taken below its one-wave threshold, or up past any batch, so the
factored route is taken above it), its launches are captured `launches` times into a CUDA graph, and the routes'
graphs are replayed alternately for `rounds` rounds, timed with CUDA events; the median per launch is reported.  Shapes: the SlowFast Fast stem (5x7x7, 3 -> 8) at batch 1, 2 and 8, on 32 frames of 224^2.
Prints the card name, power limit and max SM clock, then per route: us, GB/s of the algorithmic bytes (input + output
+ weights, f16) and the kernels launched.  Writes JSON to DIR/bench_stem.json when --out is given.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from pytorchvideo_b200 import _lib as L  # noqa: E402
from pytorchvideo_b200 import testing as TS  # noqa: E402
from pytorchvideo_b200.engine import plan as PL  # noqa: E402
from pytorchvideo_b200.engine.plan import Plan, _conv_out  # noqa: E402

# name: (batch, C_out, kernel, stride, padding)
SHAPES = {
    "fast_stem_b1": (1, 8, (5, 7, 7), (1, 2, 2), (2, 3, 3)),
    "fast_stem_b2": (2, 8, (5, 7, 7), (1, 2, 2), (2, 3, 3)),
    "fast_stem_b8": (8, 8, (5, 7, 7), (1, 2, 2), (2, 3, 3)),
}
ROUTES = {   # route: the SM count (plan.H100_SXM_SMS) the plan is built with
    "stream": 1,
    "factored": 1 << 30,
}
T, HW = 32, 224


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = "unavailable"
    return name, q


def build(shape, route, x, w, launches, dev, stream):
    """(graph of `launches` x the route's conv launches, op names, kernels launched by one run) or None when the route
    does not apply to the shape (the stream kernel below its threshold or outside its scope)."""
    _, co, k, s, p = shape
    threshold = PL.H100_SXM_SMS
    PL.H100_SXM_SMS = ROUTES[route]
    try:
        plan = Plan(dev, L.PV_F16)
        xr = plan.emit_input_ncdhw(x, 3, 4)
        plan.emit_conv(xr, w, None, None, s, p, (1, 1, 1), 1, L.ACT_RELU, None, "stem")
    finally:
        PL.H100_SXM_SMS = threshold
    conv_ops = [(n, fn) for n, fn in plan.ops if n.startswith("stem")]
    names = [n for n, _ in conv_ops]
    if (route == "stream") != (plan.stats.get("stem_stream") == 1) or names == ["stem"]:
        return None
    plan.finalize()
    with torch.cuda.stream(stream):
        plan.run(stream.cuda_stream)                 # the layout conversion, once
        stream.synchronize()
        before = TS.kernel_counts()
        for _, fn in conv_ops:
            fn(stream.cuda_stream)
        stream.synchronize()
        launched = sorted(TS.kernel_count_diff(before, TS.kernel_counts()))
        for _ in range(10):
            for _, fn in conv_ops:
                fn(stream.cuda_stream)
        stream.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            for _ in range(launches):
                for _, fn in conv_ops:
                    fn(torch.cuda.current_stream().cuda_stream)
        graph.replay()
        stream.synchronize()
    return graph, names, launched, plan


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    L.require_device()
    dev = torch.device("cuda:0")
    name, q = card()
    print("card: %s | power.limit, clocks.max.sm: %s" % (name, q), flush=True)
    res = {"card": name, "power_limit_and_max_sm_clock": q, "launches": a.launches, "rounds": a.rounds, "shapes": {}}
    stream = torch.cuda.Stream(dev)
    for sname in a.shapes.split(","):
        shape = SHAPES[sname]
        N, co, k, s, p = shape
        g = torch.Generator().manual_seed(N + co)
        x = torch.rand(N, 3, T, HW, HW, generator=g).to(dev)
        w = torch.randn(co, 3, *k, generator=g) * (2.0 / (3 * k[0] * k[1] * k[2])) ** 0.5
        To, Ho, Wo = (_conv_out(i, kk, ss, pp, 1) for i, kk, ss, pp in zip((T, HW, HW), k, s, p))
        nbytes = (N * T * HW * HW * 3 + N * To * Ho * Wo * co + w.numel()) * 2
        built = {r: build(shape, r, x, w, a.launches, dev, stream) for r in ROUTES}
        built = {r: b for r, b in built.items() if b is not None}
        times = {r: [] for r in built}
        for _ in range(a.rounds):
            for r, (graph, _, _, _) in built.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                with torch.cuda.stream(stream):
                    e0.record(stream)
                    graph.replay()
                    e1.record(stream)
                e1.synchronize()
                times[r].append(e0.elapsed_time(e1) * 1e3 / a.launches)
        out = {}
        for r, (_, names, launched, _) in built.items():
            us = statistics.median(times[r])
            out[r] = {"us": us, "us_all": times[r], "gbs": nbytes / us / 1e3, "ops": names, "kernels": launched}
            print("%-13s %-9s %9.1f us %8.0f GB/s  ops %s  kernels %s" % (sname, r, us, nbytes / us / 1e3, names,
                                                                         launched), flush=True)
        res["shapes"][sname] = {"algorithmic_bytes": nbytes, "routes": out}
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        json.dump(res, open(os.path.join(a.out, "bench_stem.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
