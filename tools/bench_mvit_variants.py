"""BatchNorm MViT-B-16x4 against LayerNorm MViT-B-16x4 on the engine: the hub geometry built with norm="batchnorm" and
with the default LayerNorm, both at one batch size.  Reports ms per step (CUDA events around graph replays, the two
models timed alternately over several rounds after a warm-up), launches per step, and the time of the attention-pool
depthwise launches of each plan (per-launch CUDA events, plan.profile): the BatchNorm plan's pools run with the
pre-activation prologue (BatchNorm3d + GELU before the pool), the LayerNorm plan's at the same shapes without it.
The card's name, power limit and SM clock are printed with the numbers.  Writes nothing.

    python tools/bench_mvit_variants.py [--batch 8] [--steps 20] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pytorchvideo_b200 import testing as TS  # noqa: E402
from pytorchvideo_b200.engine import compile_model  # noqa: E402
from pytorchvideo_b200.models import hub as H  # noqa: E402


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def _time(cm, x, steps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        cm(x)
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile-iters", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to measure")
    print("card:", _card())
    x = TS.synthetic_clip(a.batch, 16, 224, 224, seed=8).cuda()
    plans = {}
    for name, kw in (("mvit_b_16x4_batchnorm", {"norm": "batchnorm"}), ("mvit_b_16x4_layernorm", {})):
        model = H.mvit_base_16x4(**kw).eval()
        if kw:
            # builder initialisation with random BatchNorms: randomize_model's linear weights grow the residual stream
            # of a LayerNorm-free model past the f16 range (testing.MVIT_VARIANT_INIT_CASES)
            g = torch.Generator().manual_seed(3)
            with torch.no_grad():       # random BatchNorm statistics (the ranges of testing.randomize_model)
                for m in model.modules():
                    if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
                        for t, lo, hi in ((m.weight, 0.5, 1.5), (m.bias, -0.5, 0.5), (m.running_var, 0.5, 1.5),
                                          (m.running_mean, -0.5, 0.5)):
                            t.copy_(torch.rand(t.shape, generator=g) * (hi - lo) + lo)
        else:
            model = TS.randomize_model(model, seed=3).eval()
        plans[name] = compile_model(model.cuda(), x, dtype="f16")
    with torch.no_grad():
        for cm in plans.values():
            for _ in range(a.warmup):
                cm(x)
        torch.cuda.synchronize()
        times = {k: [] for k in plans}
        for _ in range(a.rounds):
            for k, cm in plans.items():
                times[k].append(_time(cm, x, a.steps))
    results = {"card": _card(), "batch": a.batch}
    for k, cm in plans.items():
        ts = sorted(times[k])
        prof = cm.plan.profile(iters=a.profile_iters)
        pools = [(n, t) for (n, _), t in zip(cm.plan.ops, prof) if ".attn.pool_" in n and n.endswith(".dwconv")]
        results[k] = {"ms_per_step_median": ts[len(ts) // 2], "ms_per_step_min": ts[0], "ms_per_step_max": ts[-1],
                      "clips_per_s": a.batch * 1000.0 / ts[len(ts) // 2], "launches_per_step": cm.plan.num_launches(),
                      "pool_launches": len(pools), "pool_ms_per_step": sum(t for _, t in pools),
                      "pool_prologue_launches": cm.plan.stats.get("pool_prologue", 0),
                      "pools_ms": {n: round(t, 4) for n, t in pools}}
    print(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
