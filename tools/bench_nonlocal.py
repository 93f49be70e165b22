"""Non-local block timings on the GPU: the I3D-NLN res3 / res4 shapes at batch 8 (8x224^2 clips).

For each shape: the wide attention kernel alone (pv_attention_fwd, q / k / v as channel slices like the lowering
feeds them), the whole engine NL block (one CUDA-graph replay), and an inline f16 ATen restatement of
NonLocal.forward (1x1x1 conv3d, max pool, einsum + softmax, conv_out + BN, residual) as the torch-gpu arm.  Then the
engine's i3d_r50 step time with and without the five NL blocks of the I3D-NLN layout.  Times are CUDA events over
``--iters`` replays after ``--warmup``; TFLOP/s of the attention uses 4 * B * Nq * Nk * D.

    python tools/bench_nonlocal.py [--iters 50] [--warmup 10]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pytorchvideo_b200 import _lib as L, testing as TS  # noqa: E402
from pytorchvideo_b200.engine import compile_model  # noqa: E402
from pytorchvideo_b200.layers.nonlocal_net import create_nonlocal  # noqa: E402

# name: (dim_in, dim_inner, input (B, C, T, H, W))
SHAPES = {"res3": (512, 256, (8, 512, 4, 28, 28)), "res4": (1024, 512, (8, 1024, 4, 14, 14))}


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


def attention_alone(B, Nq, Nk, D, iters, warmup):
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    theta = torch.randn(B, Nq, D, generator=g).half().to(dev)
    phig = torch.randn(B, Nk, 2 * D, generator=g).half().to(dev)
    o = torch.empty(B, Nq, D, dtype=torch.float16, device=dev)
    d = L.AttentionDesc()
    d.dtype, d.B, d.H, d.Nq, d.Nk, d.D = L.PV_F16, B, 1, Nq, Nk, D
    d.q_row_stride, d.k_row_stride, d.v_row_stride, d.o_row_stride = D, 2 * D, 2 * D, D
    d.q_batch_stride, d.k_batch_stride, d.v_batch_stride, d.o_batch_stride = Nq * D, Nk * 2 * D, Nk * 2 * D, Nq * D
    d.scale = D ** -0.5
    lib = L.load()
    assert lib.pv_attention_kernel_for(C.byref(d), theta.data_ptr(), phig.data_ptr(), phig.data_ptr() + 2 * D,
                                       o.data_ptr()) == L.ATTN_WIDE
    s = torch.cuda.current_stream().cuda_stream

    def run():
        L.check(lib.pv_attention_fwd(C.byref(d), theta.data_ptr(), phig.data_ptr(), phig.data_ptr() + 2 * D, o.data_ptr(), s))
    return timed(run, iters, warmup)


def torch_block(m, x):
    """f16 ATen restatement of NonLocal.forward (reference layers/nonlocal_net.py:55-94)."""
    di = m.conv_theta.out_channels
    N, Cc, T, H, W = x.shape
    theta = m.conv_theta(x)
    xp = m.pool(x) if m.pool is not None else x
    phi, g = m.conv_phi(xp).view(N, di, -1), m.conv_g(xp).view(N, di, -1)
    tp = torch.einsum("nct,ncp->ntp", (theta.view(N, di, -1), phi)) * (di ** -0.5)
    tp = F.softmax(tp, dim=2)
    y = torch.einsum("ntg,ncg->nct", (tp, g)).view(N, di, T, H, W)
    return x + m.norm(m.conv_out(y))


def i3d(nl):
    import pytorchvideo_b200.models.hub as PH
    model = PH.i3d_r50()
    if nl:
        for stage, idx in {3: (1, 3), 4: (1, 3, 5)}.items():      # res3, res4
            blocks = model.blocks[stage].res_blocks
            for i in idx:
                c = blocks[i].branch2.conv_c.out_channels
                blocks[i] = nn.Sequential(blocks[i], create_nonlocal(dim_in=c, dim_inner=c // 2, pool_size=(1, 2, 2)))
    return TS.randomize_model(model, seed=1234).eval()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    L.require_device()
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"device": torch.cuda.get_device_name(0), "nvidia_smi": smi}), flush=True)
    for name, (cin, di, shape) in SHAPES.items():
        B, _, T, H, W = shape
        Nq, Nk = T * H * W, T * (H // 2) * (W // 2)
        flops = 4.0 * B * Nq * Nk * di
        t_attn = attention_alone(B, Nq, Nk, di, a.iters, a.warmup)
        m = TS.randomize_model(create_nonlocal(dim_in=cin, dim_inner=di, pool_size=(1, 2, 2)), seed=3).eval().to(dev)
        x = torch.randn(shape, device=dev)
        cm = compile_model(m, x, dtype="f16")
        cm(x)
        t_block = timed(cm.graph.replay, a.iters, a.warmup)
        mh, xh = m.half(), x.half()
        with torch.no_grad():
            t_torch = timed(lambda: torch_block(mh, xh), a.iters, a.warmup)
            ref = torch_block(mh, xh).float()
        m.float()
        out = cm(x).float()
        rel = float((out - ref).abs().max() / ref.abs().max())
        print(json.dumps({"shape": name, "B": B, "Nq": Nq, "Nk": Nk, "D": di, "attention_ms": round(t_attn, 4),
                          "attention_tflops": round(flops / t_attn / 1e9, 1), "engine_block_ms": round(t_block, 4),
                          "torch_f16_block_ms": round(t_torch, 4), "engine_vs_torch_max_rel": rel}), flush=True)
        del cm, m, mh
        torch.cuda.empty_cache()
    clip = torch.rand(8, 3, 8, 224, 224, device=dev)
    res = {}
    for nl in (False, True):
        cm = compile_model(i3d(nl).to(dev), clip, dtype="f16")
        cm(clip)
        res["i3d_r50_b8_nl" if nl else "i3d_r50_b8"] = round(timed(cm.graph.replay, a.iters, a.warmup), 3)
        del cm
        torch.cuda.empty_cache()
    print(json.dumps({"step_ms": res}), flush=True)


if __name__ == "__main__":
    main()
