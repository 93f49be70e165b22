"""Timings of the self-supervised objectives and steps on one GPU (CUDA events, median of --iters after --warmup).

  python tools/bench_ssl.py [--iters 20] [--warmup 5]

Prints one line per measurement:
- pv_memory_bank_ce at B = 64, neg_size = 4096 with dim 128 and 2048: time and achieved GB/s, counting
  B * (K + 1) * dim * 4 bytes of gathered bank rows plus the int64 indices;
- a BYOL step on the Slow-R50 case of tests/golden/ssl.pt (batch 2 of 8 x 224^2), split into the online plan, the EMA
  update, the in-place refresh of the momentum plan (against compiling it again), its replay and the loss;
- a SimCLR step on the same trunk and projector.
"""
import argparse
import os
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pytorchvideo_b200 import config, contrastive as K, testing as TS  # noqa: E402
from pytorchvideo_b200.engine import lower as _lower  # noqa: E402
from pytorchvideo_b200.layers import make_multilayer_perceptron  # noqa: E402
from pytorchvideo_b200.models.byol import BYOL  # noqa: E402
from pytorchvideo_b200.models.memory_bank import MemoryBank  # noqa: E402
from pytorchvideo_b200.models.resnet import create_resnet  # noqa: E402
from pytorchvideo_b200.models.simclr import SimCLR  # noqa: E402

NS = types.SimpleNamespace(SimCLR=SimCLR, BYOL=BYOL, MemoryBank=MemoryBank, create_resnet=create_resnet,
                           make_multilayer_perceptron=make_multilayer_perceptron)


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    dev = "cuda"
    print("device:", torch.cuda.get_device_name(0))
    B, K1, bank = 64, 4097, 1280000
    for dim in (128, 2048):
        rows = bank if dim == 128 else 200000
        mem = torch.rand((rows, dim), device=dev)
        x = K.l2_normalize(torch.randn((B, dim), device=dev))
        idx = torch.randint(0, rows, (B, K1), device=dev)
        ms = timed(lambda: K.memory_bank_ce(x, mem, idx, 0.07), a.iters, a.warmup)
        nbytes = B * K1 * dim * 4 + B * K1 * 8
        print("memory_bank_ce B=%d K=%d dim=%d bank=%d: %.3f ms  %.0f GB/s (of 3350)" % (B, K1, dim, rows, ms,
                                                                                         nbytes / ms / 1e6))
        del mem
    m, (x1, x2) = TS.build_ssl_case("byol_video", NS)
    m = m.to(dev)
    x1, x2 = x1.to(dev), x2.to(dev)
    m(x1, x2)
    st = m._state()
    print("byol online plan:   %.3f ms" % timed(lambda: st["online"].embed(x1), a.iters, a.warmup))
    print("byol ema update:    %.3f ms" % timed(lambda: st["ema"](m.mmt), a.iters, a.warmup))

    (cm, refresh), = st["plans"].values()
    print("byol momentum plan refresh (pv_weights_refresh): %.3f ms" % timed(refresh, a.iters, a.warmup))

    def recompile():
        c = _lower.compile_model(st["mmt"], x1, config.get_precision(), config.get_use_graph())
        c(x1)
    print("byol momentum plan compiled again instead: %.3f ms" % timed(recompile, max(3, a.iters // 4), 1))
    print("byol momentum plan, replay:         %.3f ms" % timed(lambda: m._mmt_embed(x1), a.iters, a.warmup))
    q = K.l2_normalize(torch.randn((4, 128), device=dev))
    print("byol loss:          %.3f ms" % timed(lambda: K.contrastive_ce(q, q, 1.0, 0, True), a.iters, a.warmup))
    print("byol step:          %.3f ms" % timed(lambda: m(x1, x2), max(3, a.iters // 4), 1))
    s, (y1, y2) = TS.build_ssl_case("simclr_video", NS)
    s = s.to(dev)
    y1, y2 = y1.to(dev), y2.to(dev)
    print("simclr step:        %.3f ms" % timed(lambda: s(y1, y2), a.iters, a.warmup))


if __name__ == "__main__":
    main()
