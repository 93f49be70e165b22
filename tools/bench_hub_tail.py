"""The image MViT-B-16 and SlowFast-16x8-R101-50-50 hub entries on the engine: ms per step (and images/s) of the image
MViT at one batch size and of the SlowFast at another, and every distinct attention pool of the image MViT on the plane
kernel (pv_dwplane_fwd) against the route pv_dwconv3d_fwd takes for it (its tile kernel or the generic stencil).
Models are timed with CUDA events around graph replays after a warm-up, several rounds; the pools alternate the two
kernels round by round and report the median.  The card's name, power limit and SM clock are printed with the numbers.
Writes nothing.

    python tools/bench_hub_tail.py [--mvit-batch 64] [--slowfast-batch 8] [--steps 20] [--rounds 5]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pytorchvideo_b200 import _lib as L  # noqa: E402
from pytorchvideo_b200 import testing as TS  # noqa: E402
from pytorchvideo_b200.models import hub as H  # noqa: E402

# the image MViT's pools at 224^2: (plane, stride, pooled channels, token row stride, channel offset, what)
POOLS = [
    (56, 4, 192, 288, 96, "block 0 K|V"),
    (56, 2, 96, 288, 0, "block 1 pool_q"),
    (28, 2, 384, 576, 192, "blocks 1-2 K|V"),
    (28, 2, 192, 576, 0, "block 3 pool_q"),
    (14, 1, 768, 1152, 384, "blocks 3-13 K|V"),
    (14, 2, 384, 1152, 0, "block 14 pool_q"),
    (7, 1, 1536, 2304, 768, "blocks 14-15 K|V"),
]


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def _events(fn, reps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / reps


def _model(name, x, a):
    m = TS.randomize_model(getattr(H, name)(), seed=5).eval().cuda()
    with torch.no_grad():
        for _ in range(a.warmup):
            m(x)
        torch.cuda.synchronize()
        ts = sorted(_events(lambda: m(x), a.steps) for _ in range(a.rounds))
    m.cpu()
    return ts


def _pool(N, H_, s, C, rs, off, a):
    Ho = (H_ + 2 - 3) // s + 1
    x = torch.randn(N, 1 + H_ * H_, rs, device="cuda").half()
    y = torch.empty(N, 1 + Ho * Ho, C, device="cuda", dtype=torch.float16)
    w = (torch.randn(9, C, device="cuda") * 0.3).half()
    one, zero = torch.ones(C, device="cuda"), torch.zeros(C, device="cuda")
    d = L.Conv3dDesc()
    d.dtype, d.N, d.Ti, d.Hi, d.Wi, d.Ci = L.PV_F16, N, 1, H_, H_, C
    d.To, d.Ho, d.Wo, d.Co = 1, Ho, Ho, C
    d.kt, d.kh, d.kw, d.st, d.sh, d.sw, d.pt, d.ph, d.pw, d.dt, d.dh, d.dw = 1, 3, 3, 1, s, s, 0, 1, 1, 1, 1, 1
    d.groups, d.x_row_stride, d.y_row_stride = C, rs, C
    d.x_batch_stride, d.y_batch_stride = (1 + H_ * H_) * rs, (1 + Ho * Ho) * C
    lib, stream = L.load(), torch.cuda.current_stream().cuda_stream
    xp, yp = x.data_ptr() + (rs + off) * 2, y.data_ptr() + C * 2
    routes = {
        "plane": lambda: L.check(lib.pv_dwplane_fwd(ctypes.byref(d), xp, w.data_ptr(), one.data_ptr(), zero.data_ptr(),
                                                    yp, stream), "pv_dwplane_fwd"),
        "before": lambda: L.check(lib.pv_dwconv3d_fwd(ctypes.byref(d), xp, w.data_ptr(), one.data_ptr(), zero.data_ptr(),
                                                      yp, None, stream), "pv_dwconv3d_fwd"),
    }
    kernels = {}
    for k, fn in routes.items():
        _, ran = TS.launched_kernels(fn)
        kernels[k] = sorted(ran)
        for _ in range(a.warmup):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in routes}
    for _ in range(a.rounds):
        for k, fn in routes.items():
            times[k].append(_events(fn, a.pool_reps))
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    nbytes = (N * H_ * H_ + N * Ho * Ho) * C * 2
    return {"plane_us": med["plane"] * 1e3, "before_us": med["before"] * 1e3, "before_kernel": kernels["before"],
            "plane_kernel": kernels["plane"], "speedup": med["before"] / med["plane"],
            "plane_GBps": nbytes / (med["plane"] * 1e-3) / 1e9}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mvit-batch", type=int, default=64)
    ap.add_argument("--slowfast-batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--pool-reps", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to measure")
    print("card:", _card())
    res = {}
    ts = _model("mvit_base_16", TS.synthetic_clip(a.mvit_batch, 1, 224, 224, seed=8)[:, :, 0].contiguous().cuda(), a)
    res["mvit_base_16"] = {"batch": a.mvit_batch, "ms_per_step_median": ts[len(ts) // 2], "ms_per_step_min": ts[0],
                           "ms_per_step_max": ts[-1], "images_per_s": a.mvit_batch * 1000.0 / ts[len(ts) // 2]}
    x = [t.cuda() for t in TS.slowfast_inputs(TS.synthetic_clip(a.slowfast_batch, 64, 224, 224, seed=8))]
    ts = _model("slowfast_16x8_r101_50_50", x, a)
    res["slowfast_16x8_r101_50_50"] = {"batch": a.slowfast_batch, "ms_per_step_median": ts[len(ts) // 2],
                                       "ms_per_step_min": ts[0], "ms_per_step_max": ts[-1]}
    del x
    res["pools"] = {"%s (%dx%d s%d, %d ch)" % (what, p, p, s, c): _pool(a.mvit_batch, p, s, c, rs, off, a)
                    for p, s, c, rs, off, what in POOLS}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
