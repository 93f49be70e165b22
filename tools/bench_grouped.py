"""Grouped convolutions on the H100: grouped mode of the TMA-fed kernel against the dense expansion.

    python tools/bench_grouped.py [--batch 8] [--launches 200] [--runs 3] [--out DIR]

Prints the card name and power limit, then
  (1) per layer: every distinct grouped conv_b shape of slow_r50_g32, csn_r101_w8 and slowfast_r50_g (testing.
      GROUPED_MODEL_CASES) at the given batch, as the grouped-mode launch and as the dense convolution of the
      block-diagonal weights, each timed with CUDA events over `launches` launches replayed from a CUDA graph after a
      warm-up, with the tensor-core multiply-adds each does;
  (2) whole model: the resident step time (CUDA-graph replay, inputs on the device) of slow_r50 with 32 groups against
      the dense slow_r50 at the same batch, `runs` alternating runs of each.
Writes the result as JSON to DIR/bench_grouped.json when --out is given.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from pytorchvideo_b200 import _lib as L  # noqa: E402
from pytorchvideo_b200 import testing as TS  # noqa: E402
from pytorchvideo_b200.engine import packing as PK  # noqa: E402
from pytorchvideo_b200.engine.plan import Plan  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = "unavailable"
    return name, q


def grouped_shapes(batch):
    """Distinct (C, groups, kernel, stride, padding, dilation, T, H, W) of the grouped (not depthwise) convolutions of
    the three grouped model cases, recorded from a host-side lowering at batch 1."""
    import pytorchvideo_b200.models.hub as PH
    from pytorchvideo_b200.engine.lower import lower_only
    shapes = {}
    orig = Plan.emit_conv
    for case in ("slow_r50_g32", "csn_r101_w8", "slowfast_r50_g"):
        hub, kw, _, T, H, W, is_sf, _ = TS.GROUPED_MODEL_CASES[case]
        model = getattr(PH, hub)(**kw).eval()
        seen = []

        def rec(self, x, weight, conv_bias, bn, stride, padding, dilation, groups, *args, **kwargs):
            if 1 < groups and not groups == weight.shape[0] == x.C:
                seen.append((x.C, groups, tuple(weight.shape[2:]), tuple(stride), tuple(padding), tuple(dilation),
                             x.T, x.H, x.W))
            return orig(self, x, weight, conv_bias, bn, stride, padding, dilation, groups, *args, **kwargs)
        Plan.emit_conv = rec
        try:
            clip = torch.zeros(1, 3, T, H, W)
            lower_only(model, TS.slowfast_inputs(clip) if is_sf else clip)
        finally:
            Plan.emit_conv = orig
        for s in seen:
            shapes.setdefault(s, set()).add(case)
    return sorted(shapes.items())


def time_conv(shape, batch, expand, launches, dev):
    C, groups, k, s, p, dil, T, H, W = shape
    g = torch.Generator().manual_seed(C + groups)
    w = torch.randn(C, C // groups, *k, generator=g) * (2.0 / (C // groups * k[0] * k[1] * k[2])) ** 0.5
    x = torch.rand(batch, C, T, H, W, generator=g).to(dev)
    plan = Plan(dev, L.PV_F16)
    xr = plan.emit_input_ncdhw(x, C, C)
    plan.materialize_input(xr)
    n0 = len(plan.ops)
    if expand:
        y = plan.emit_conv(xr, PK.expand_grouped_dense(w, groups), None, None, s, p, dil, 1, L.ACT_RELU, None, "conv")
    else:
        y = plan.emit_conv(xr, w, None, None, s, p, dil, groups, L.ACT_RELU, None, "conv")
    assert len(plan.ops) == n0 + 1
    kind = plan.meta[n0]["kind"]
    plan.finalize()
    stream = torch.cuda.Stream(dev)
    fn = plan.ops[n0][1]
    with torch.cuda.stream(stream):
        plan.run(stream.cuda_stream)                         # the layout conversion and one warm-up launch
        for _ in range(20):
            fn(stream.cuda_stream)
        stream.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            for _ in range(launches):
                fn(torch.cuda.current_stream().cuda_stream)
        graph.replay()
        stream.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        graph.replay()
        e1.record(stream)
        e1.synchronize()
    ms = e0.elapsed_time(e1) / launches
    To, Ho, Wo = ((i + 2 * pp - d * (kk - 1) - 1) // ss + 1 for i, kk, ss, pp, d in zip((T, H, W), k, s, p, dil))
    m = batch * To * Ho * Wo
    taps = k[0] * k[1] * k[2]
    if expand:
        macs = m * taps * PK.pad_to(C, 64) * C
    else:
        _, _, span_k, _ = L.group_span(plan._conv_desc(xr, (To, Ho, Wo), C, k, s, p, dil, groups, L.ACT_RELU, None, C, 0))
        macs = m * taps * span_k * C
    return ms, macs, kind


def model_step(hub_kwargs, batch, dev, steps=20):
    import pytorchvideo_b200.models.hub as PH
    from pytorchvideo_b200.engine import compile_model
    model = TS.randomize_model(PH.slow_r50(**hub_kwargs), seed=1234, f16_weights=True).eval()
    clip = TS.synthetic_clip(batch, 8, 224, 224, seed=42, f16_values=True).to(dev)
    cm = compile_model(model, clip, dtype="f16", use_graph=True)
    for _ in range(5):
        cm(clip)
    torch.cuda.synchronize()

    def run():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(steps):
            cm(clip)
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / steps
    return run, cm.plan.stats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    L.require_device()
    dev = torch.device("cuda:0")
    name, q = card()
    print("card: %s | power.limit, clocks.max.sm: %s" % (name, q), flush=True)
    res = {"card": name, "power_limit_and_max_sm_clock": q, "batch": a.batch, "layers": [], "model": {}}
    print("%-44s %-28s %10s %10s %8s %9s %9s" % ("layer (C/groups, k, s, in T,H,W)", "models", "grouped ms", "dense ms",
                                                  "speedup", "g GMAC", "d GMAC"))
    for shape, cases in grouped_shapes(a.batch):
        C, groups, k, s, p, dil, T, H, W = shape
        label = "%d/%d k%s s%s %dx%dx%d" % (C, groups, "".join(map(str, k)), "".join(map(str, s)), T, H, W)
        td, md, kd = time_conv(shape, a.batch, True, a.launches, dev)
        tg, mg, kg = time_conv(shape, a.batch, False, a.launches, dev)
        if kg != "grouped":            # one group span: the layer runs as the dense expansion anyway
            print("%-44s %-28s %10s %10.4f %8s %9s %9.2f  (%s)" % (label, ",".join(sorted(cases)), "-", td, "-", "-",
                                                                  md / 1e9, kd), flush=True)
            res["layers"].append({"shape": list(map(str, shape)), "models": sorted(cases), "dense_ms": td,
                                  "dense_kind": kd, "dense_macs": md, "note": "one span: runs expanded"})
            continue
        print("%-44s %-28s %10.4f %10.4f %8.2f %9.2f %9.2f  (%s / %s)" % (label, ",".join(sorted(cases)), tg, td, td / tg,
                                                                       mg / 1e9, md / 1e9, kg, kd), flush=True)
        res["layers"].append({"shape": list(map(str, shape)), "models": sorted(cases), "grouped_ms": tg, "dense_ms": td,
                              "grouped_kind": kg, "dense_kind": kd, "grouped_macs": mg, "dense_macs": md})
    runs = {"slow_r50_g32": [], "slow_r50": []}
    run_g, stats_g = model_step({"stage_conv_b_num_groups": (32,) * 4}, a.batch, dev)
    run_d, stats_d = model_step({}, a.batch, dev)
    for _ in range(a.runs):
        runs["slow_r50_g32"].append(run_g())
        runs["slow_r50"].append(run_d())
    for k_, v in runs.items():
        print("resident step %-14s batch %d: %s ms" % (k_, a.batch, " / ".join("%.3f" % t for t in v)), flush=True)
    res["model"] = {"runs_ms": runs, "stats": {"slow_r50_g32": stats_g, "slow_r50": stats_d}}
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        json.dump(res, open(os.path.join(a.out, "bench_grouped.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
