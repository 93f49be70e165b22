"""Masked multistream timings on the GPU at batch 32 with random ragged lengths (seeded).

Three shapes: a bidirectional LSTM (dim_in 2048, hidden 512, T 128), TransposeMultiheadAttention (512 features,
8 heads, T 128) and TransposeTransformerEncoder (512 wide, 8 heads, 2 layers, T 128).  Each runs as the engine module
(f16, one CUDA-graph replay per call) and as an f16 torch-GPU arm on the same inputs doing what the reference's
forward does: cuDNN nn.LSTM over pack_padded_sequence, nn.MultiheadAttention with need_weights=True and a key padding
mask, nn.TransformerEncoder with a key padding mask.  Times are CUDA events over ``--iters`` calls after ``--warmup``;
the LSTM line also gives the engine's recurrence launch alone (Plan.profile) per step.  The card's name and power limit
are printed with the numbers.

    python tools/bench_masked.py [--iters 50] [--warmup 10]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn as nn
from torch.nn.utils.rnn import pack_padded_sequence

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pytorchvideo_b200.models import LSTM, TransposeMultiheadAttention, TransposeTransformerEncoder  # noqa: E402

B, T = 32, 128


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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
    except Exception:        # noqa: BLE001 - the numbers stay valid without the label
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def inputs(F, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, F, generator=g)
    lengths = torch.randint(1, T + 1, (B,), generator=g)
    mask = torch.arange(T)[None, :] < lengths[:, None]
    return x.cuda(), mask.cuda()


def bench_lstm(iters, warmup):
    x, mask = inputs(2048)
    m = LSTM(2048, 512, bidirectional=True).cuda().eval()
    ref = nn.LSTM(2048, 512, batch_first=True, bidirectional=True).cuda().half().eval()
    ref.load_state_dict({k: v.half() for k, v in m.lstm.state_dict().items()})
    xh = x.half()

    def torch_arm():
        packed = pack_padded_sequence(xh, mask.sum(1).clamp(1, T).cpu(), batch_first=True, enforce_sorted=False)
        _, (h, _) = ref(packed)
        return torch.cat([h[0], h[1]], -1)
    with torch.no_grad():
        eng = timed(lambda: m(x, mask), iters, warmup)
        tor = timed(torch_arm, iters, warmup)
        diff = float((m(x, mask).float() - torch_arm().float()).abs().max())
        cm = next(iter(m.__dict__["_pv_cache"].values()))
        prof = cm.plan.profile(iters=10)
        rec = sum(t for t, meta in zip(prof, cm.plan.meta) if meta["name"].endswith("recurrence"))
    return {"shape": "lstm_bi dim_in 2048 H 512", "engine_ms": eng, "torch_f16_ms": tor, "recurrence_ms": rec,
            "recurrence_us_per_step": rec * 1000.0 / T, "max_abs_diff": diff}


def bench_mha(iters, warmup):
    x, mask = inputs(512, seed=1)
    m = TransposeMultiheadAttention(512, 8).cuda().eval()
    ref = nn.MultiheadAttention(512, 8).cuda().half().eval()
    ref.load_state_dict({k: v.half() for k, v in m._attention.state_dict().items()})
    xt = x.half().transpose(0, 1)

    def torch_arm():
        kpm = mask.clone()
        kpm[:, 0] = True
        return ref(xt, xt, xt, key_padding_mask=~kpm)[0].transpose(0, 1)
    with torch.no_grad():
        eng = timed(lambda: m(x, mask), iters, warmup)
        tor = timed(torch_arm, iters, warmup)
        diff = float((m(x, mask).float() - torch_arm().float()).abs().max())
    return {"shape": "mha F 512 heads 8", "engine_ms": eng, "torch_f16_ms": tor, "max_abs_diff": diff}


def bench_encoder(iters, warmup):
    x, mask = inputs(512, seed=2)
    m = TransposeTransformerEncoder(512, 8, 2).cuda().eval()
    ref = nn.TransformerEncoder(nn.TransformerEncoderLayer(512, 8), 2).cuda().half().eval()
    ref.load_state_dict({k: v.half() for k, v in m.encoder.state_dict().items()})
    xt = x.half().transpose(0, 1)

    def torch_arm():
        kpm = mask.clone()
        kpm[:, 0] = True
        return ref(src=xt, src_key_padding_mask=~kpm).transpose(0, 1)[:, 0, :]
    with torch.no_grad():
        eng = timed(lambda: m(x, mask), iters, warmup)
        tor = timed(torch_arm, iters, warmup)
        diff = float((m(x, mask).float() - torch_arm().float()).abs().max())
    return {"shape": "encoder 512 heads 8 layers 2", "engine_ms": eng, "torch_f16_ms": tor, "max_abs_diff": diff}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_masked.py needs a GPU")
    name, power = card()
    print("card: %s, power limit %s, B %d, T %d" % (name, power, B, T))
    for fn in (bench_lstm, bench_mha, bench_encoder):
        r = fn(a.iters, a.warmup)
        r.update(card=name, power_limit=power)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
