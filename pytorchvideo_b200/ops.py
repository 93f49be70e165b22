"""Eager single-op entry points (NCDHW torch tensors in/out) built on the same Plan emitters the
compiled models use.  Mainly for tests and for users who want one fused op without a model."""
import ctypes as C

import torch

from . import _lib as L
from .engine.plan import Plan, TRef

_DT = {"f16": L.PV_F16, "f32": L.PV_F32}
_ACT = {None: L.ACT_NONE, "none": L.ACT_NONE, "relu": L.ACT_RELU, "swish": L.ACT_SWISH, "gelu": L.ACT_GELU,
        "sigmoid": L.ACT_SIGMOID}


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


def _require_cuda(*ts):
    L.require_device()
    for t in ts:
        if t is not None and t.device.type != "cuda":
            raise RuntimeError("pytorchvideo_b200 ops need CUDA tensors (no CPU path)")


def conv3d_bn_act(x, weight, bias=None, bn=None, stride=(1, 1, 1), padding=(0, 0, 0), dilation=(1, 1, 1),
                  groups=1, act=None, residual=None, dtype="f16", algo=None, se_sums=False):
    """y = act(BN(conv3d(x)) + residual); x, residual: [N,C,T,H,W] CUDA tensors; returns f32 NCDHW.
    se_sums=True (depthwise): stats additionally carries "se_sums" = per-(n, c) output sums [N, C]."""
    _require_cuda(x, residual)
    plan = Plan(x.device, _DT[dtype])
    xin = x.contiguous().float()
    xr = plan.emit_input_ncdhw(xin, x.shape[1], 4 if x.shape[1] <= 4 else (x.shape[1] + 7) // 8 * 8)
    rr = None
    if residual is not None:
        rin = residual.contiguous().float()
        rr = plan.emit_input_ncdhw(rin, residual.shape[1], (residual.shape[1] + 7) // 8 * 8)
    force = {None: None, "direct": L.ALGO_DIRECT, "tcgen05": L.ALGO_TCGEN05}[algo]
    y = plan.emit_conv(xr, weight, bias, bn, tuple(stride), tuple(padding), tuple(dilation), groups, _ACT[act], rr,
                       "conv", force_algo=force, se_sums=se_sums)
    out, shape = plan.emit_to_ncdhw(y)
    plan.finalize()
    plan.run(_stream(x.device))
    torch.cuda.synchronize(x.device)
    stats = dict(plan.stats)
    if se_sums:
        # int64 fixed point (2^-24) per (sample, channel), see se_sum_add in csrc/pv_common.cuh
        stats["se_sums"] = (y.se_sums.tensor.view(torch.int64).view(x.shape[0], -1)[:, : weight.shape[0]].double() / 2 ** 24).float()
    return out.tensor[: int(torch.tensor(shape).prod())].view(*shape).clone(), stats


def pool3d(x, mode, kernel, stride, padding, dtype="f16"):
    _require_cuda(x)
    plan = Plan(x.device, _DT[dtype])
    xr = plan.emit_input_ncdhw(x.contiguous().float(), x.shape[1], (x.shape[1] + 7) // 8 * 8)
    y = plan.emit_pool(xr, L.POOL_MAX if mode == "max" else L.POOL_AVG, tuple(kernel), tuple(stride), tuple(padding))
    out, shape = plan.emit_to_ncdhw(y)
    plan.finalize()
    plan.run(_stream(x.device))
    torch.cuda.synchronize(x.device)
    return out.tensor[: int(torch.tensor(shape).prod())].view(*shape).clone()


def roi_align(x, boxes, output_size, spatial_scale, sampling_ratio=0, dtype="f16"):
    """torchvision-style RoIAlign (aligned=False) of a [N, C, H, W] CUDA feature map for [K, 5] boxes
    (batch index, x1, y1, x2, y2) -> [K, C, ph, pw] fp32 (pv_roi_align_fwd)."""
    _require_cuda(x)
    plan = Plan(x.device, _DT[dtype])
    x5 = x.contiguous().float().unsqueeze(2)
    xr = plan.emit_input_ncdhw(x5, x5.shape[1], (x5.shape[1] + 7) // 8 * 8)
    rois = plan.raw_input(boxes.to(x.device).float().contiguous())
    osz = (output_size, output_size) if isinstance(output_size, int) else tuple(output_size)
    y = plan.emit_roi_align(xr, rois, osz, spatial_scale, sampling_ratio)
    out, shape = plan.emit_to_ncdhw(y)
    plan.finalize()
    plan.run(_stream(x.device))
    torch.cuda.synchronize(x.device)
    return out.tensor[: int(torch.tensor(shape).prod())].view(*shape).squeeze(2).clone()


def layernorm(x, gamma, beta, eps=1e-6, dtype="f16"):
    """LayerNorm over the last dim of a [rows, C] CUDA tensor (C % 8 == 0)."""
    _require_cuda(x)
    lib = L.load()
    tdt = torch.float16 if dtype == "f16" else torch.float32
    xs = x.to(tdt).contiguous()
    y = torch.empty_like(xs)
    g, b = gamma.float().contiguous().to(x.device), beta.float().contiguous().to(x.device)
    rows, Cc = xs.shape
    L.check(lib.pv_layernorm(xs.data_ptr(), y.data_ptr(), _DT[dtype], rows, 1, Cc, Cc, Cc, g.data_ptr(), b.data_ptr(),
                             float(eps), _stream(x.device)), "pv_layernorm")
    torch.cuda.synchronize(x.device)
    return y.float()


def add_layernorm(a, b, gamma, beta, eps=1e-6):
    """fp32-trunk residual add + LayerNorm: a [rows, C] (f16 or f32 CUDA tensor, used as is), b [rows, C] f16 or None.
    Returns (a + b as f32, LayerNorm(a + b) as f16)."""
    _require_cuda(a)
    lib = L.load()
    a = a.contiguous()
    assert a.dtype in (torch.float16, torch.float32)
    bb = None if b is None else b.half().contiguous()
    rows, Cc = a.shape
    s = torch.empty((rows, Cc), dtype=torch.float32, device=a.device)
    y = torch.empty((rows, Cc), dtype=torch.float16, device=a.device)
    g, be = gamma.float().contiguous().to(a.device), beta.float().contiguous().to(a.device)
    L.check(lib.pv_add_layernorm(a.data_ptr(), _DT["f16" if a.dtype == torch.float16 else "f32"], Cc,
                                 None if bb is None else bb.data_ptr(), Cc, s.data_ptr(), Cc, y.data_ptr(), Cc, rows, Cc,
                                 g.data_ptr(), be.data_ptr(), float(eps), _stream(a.device)), "pv_add_layernorm")
    torch.cuda.synchronize(a.device)
    return s, y


def attention(q, k, v, scale, add_q_residual=False, dtype="f16"):
    """q: [B,H,Nq,D], k/v: [B,H,Nk,D] CUDA tensors -> [B,H,Nq,D] (f32)."""
    _require_cuda(q, k, v)
    lib = L.load()
    tdt = torch.float16 if dtype == "f16" else torch.float32
    B, H, Nq, D = q.shape
    Nk = k.shape[2]
    # kernel layout: [B][N][H][D]
    qs = q.permute(0, 2, 1, 3).contiguous().to(tdt)
    ks = k.permute(0, 2, 1, 3).contiguous().to(tdt)
    vs = v.permute(0, 2, 1, 3).contiguous().to(tdt)
    o = torch.empty_like(qs)
    d = L.AttentionDesc()
    d.dtype, d.B, d.H, d.Nq, d.Nk, d.D = _DT[dtype], B, H, Nq, Nk, D
    d.q_row_stride = d.k_row_stride = d.v_row_stride = d.o_row_stride = H * D
    d.q_batch_stride = d.o_batch_stride = Nq * H * D
    d.k_batch_stride = d.v_batch_stride = Nk * H * D
    d.scale, d.add_q_residual = float(scale), 1 if add_q_residual else 0
    L.check(lib.pv_attention_fwd(C.byref(d), qs.data_ptr(), ks.data_ptr(), vs.data_ptr(), o.data_ptr(),
                                 _stream(q.device)), "pv_attention_fwd")
    torch.cuda.synchronize(q.device)
    return o.permute(0, 2, 1, 3).float()
