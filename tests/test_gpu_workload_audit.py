"""Every launch of the seven bench.py workloads against float64, at the shapes the benchmark runs.

The kernel matrices test each compiled instance on small synthetic shapes.  This file checks the launches the
benchmark actually makes: concat buffers written through retargeted TRefs, Block-N choices at real M, long persistent
tile walks, the window-mode and stem-stream inputs at 224^2, SE sums at batch 32 and the fp32 MViT trunk.  Each op
of a plan carries a record of what it computes (``Plan.op_spec``); the audit walks the plan on one stream, reads each
op's inputs just before it runs (so in-place ops are checked against their own operands, and errors do not compound
from op to op), runs it, asserts that the launched instances belong to the family the record implies, and compares
the output with the same operation in float64 on the GPU under the bounds of the kernel matrices (conv, fused block
and attention bounds of testing.py, the CUDA-core bounds of test_gpu_simt_matrix.py; bit-exact for layout
conversions, max pooling, copies and add_pos_cls).  Pad channels of every output must be zero, and channels of a
shared concat buffer outside the op's slice must be left as they were.

The kernels run the full batch.  The reference and the comparison cover clips 0, B // 2 and B - 1: eval forward has
no coupling between clips, and the three clips cover the first tiles, the last (ragged) tiles and the middle of
every launch's tile walk while keeping the float64 copies (moved to the host for the comparison) to a few minutes
for the file.

After the audit, the same plan is captured as the benchmark runs it (several lanes on side streams, PDL, one CUDA
graph) and replayed; every plan buffer must equal the single-stream run bit for bit, also after a replay on other
inputs (a lane reading a buffer before its producer finished would see the other input's values).

CPU tests: every launch of every workload has a record the audit checks, the read / write declarations that order
the lanes cover every buffer a record reads and writes, and sampled records agree with their torch modules.

Measured on an NVIDIA H100 80GB HBM3 (700 W power limit): 748 of the 778 launches audited (the other 30 are the
SE-sum clears of the two X3D plans, which compute no value).  Largest err / tol per family over the seven workloads:
conv igemm / gather / stem 0.996, depthwise 0.996, fused block 0.581, stem stream 0.857, temporal tap sum 0.989, average pool 0.980, scale_act
0.999, se_gate 0.005, head 0.010, LayerNorm 0.985 / 0.986 (sets), add_layernorm 0.986, attention 0.218, MViT
pooling conv 0.996; layout conversions, max pooling, copies, add_pos_cls and the add_layernorm sums bit-exact.  Graph
replay equal to the single-stream run in every buffer of every workload.  The file took 5.5 minutes (csn_r101 86 s,
mvit_base_16x4 71 s, r2plus1d_r50 53 s, slowfast_r50 43 s, x3d_m 29 s, slow_r50 26 s, x3d_xs 3 s, plus set-up).
"""
import math
import os
import sys
import time

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from pytorchvideo_b200 import _lib as L  # noqa: E402
from pytorchvideo_b200 import testing as TS  # noqa: E402
from pytorchvideo_b200.engine import packing as PK  # noqa: E402
from pytorchvideo_b200.engine.plan import Buf, TRef  # noqa: E402

WORKLOADS = sorted(bench.WORKLOADS)
# ops that produce no value of their own: the clear of a depthwise conv's SE-sum accumulator
NO_VALUE_SUFFIXES = (".se_zero",)

ACT_NAME = {L.ACT_NONE: "none", L.ACT_RELU: "relu", L.ACT_SWISH: "swish", L.ACT_GELU: "gelu",
            L.ACT_SIGMOID: "sigmoid", L.ACT_HSWISH: "hswish"}

_TC = ("conv3d_igemm_kernel<", "conv3d_igemm_gather_kernel<", "conv3d_igemm_grouped_kernel<",
       "conv3d_stem_rows_kernel<", "conv3d_stem_stream_kernel<")
_DW = ("dwconv3d_lane_kernel<", "dwconv_temporal_kernel<", "dwconv3d_tile_kernel<", "dwconv_plane_kernel<",
       "dwconv3d_kernel<", "dwconv3d_w4_kernel<")
_LN = ("layernorm_reg_kernel", "layernorm_kernel")
_ATTN = ("attention_wgmma_kernel<", "attention_mma_kernel<", "attention_kernel<", "attention_wide_kernel<",
         "attention_wide_simt_kernel<")
# instance families a record's launch may take, by record kind (conv: by route)
FAMILY = {
    "tcgen05": _TC, "grouped": _TC, "stem_stream": _TC, "direct": ("conv3d_direct_kernel<",),
    "depthwise": _DW + ("channel_sum_kernel",), "token_conv": _DW,
    "to_ndhwc": ("ncdhw_to_ndhwc_kernel", "ncdhw_to_ndhwc_padw_kernel", "ncdhw_f32_to_ndhwc4_padw_kernel"),
    "tap_sum": ("temporal_tap_sum_kernel",), "fused_block": ("bottleneck_fused_kernel<",),
    "pool": ("pool3d_kernel", "global_pool_kernel"), "head_reduce": ("head_reduce_kernel",),
    "se_gate": ("se_gate_kernel",), "scale_act": ("scale_act_kernel",), "pos_cls": ("add_pos_cls_kernel",),
    "layernorm": _LN + ("add_layernorm_kernel",), "layernorm_sets": _LN, "add_layernorm": ("add_layernorm_kernel",),
    "attention": _ATTN, "copy_cls": ("copy_rows_kernel",),
}


def supported(spec):
    """True when the audit has a reference for this record."""
    if spec is None:
        return False
    k = spec["kind"]
    if k == "conv":
        return spec["route"] in FAMILY
    if k == "token_conv":
        return not spec["prologue"]
    if k == "attention":
        return spec["normalize"] == 0
    return k in FAMILY


def family_of(spec):
    return FAMILY[spec["route"] if spec["kind"] == "conv" else spec["kind"]]


def record_io(spec):
    """(plan tensors the op reads, plan tensors it writes) according to its record."""
    k = spec["kind"]
    if k == "conv":
        ins = [spec["x"]] + [t for t in (spec["residual"],) if t is not None]
        if spec["addend"] is not None:
            ins.append(spec["addend"][0])
        return ins, [spec["y"]] + ([spec["se_sums"]] if spec["se_sums"] is not None else [])
    if k == "to_ndhwc":
        return [], [spec["y"]]
    if k in ("head_reduce", "to_f32"):
        return [spec["x"]], [spec["out"]]
    if k == "se_gate":
        return [spec["sums"]], [spec["gate"]]
    if k == "channel_sum":
        return [spec["x"]], [spec["sums"]]
    if k == "scale_act":
        return [spec["x"]] + ([spec["gate"]] if spec["gate"] is not None else []), [spec["y"]]
    if k == "add_layernorm":
        return [spec["a"], spec["br"]], [t for t in (spec["s"], spec["y"]) if t is not None]
    if k == "layernorm_sets":
        return [spec["x"], spec["y"]], [spec["y"]]
    if k == "attention":
        return [spec["q"], spec["k"], spec["v"]], [spec["o"]]
    return [spec["x"]], [spec["y"]]


def _bufs(items):
    return {id(t if isinstance(t, Buf) else t.buf) for t in items if t is not None and
            (isinstance(t, Buf) or t.buf is not None)}


# =====================================================================================================================
# reading plan tensors
# =====================================================================================================================
def full_rows(t):
    """[N, T, H, W, row_stride] view of the whole rows a TRef lives in (W-padded stem inputs: their visible columns)."""
    b = t.buf.tensor
    if t.padw is not None:
        wp, wphys = t.padw
        return b[:t.N * t.T * t.H * wphys * t.Cp].view(t.N, t.T, t.H, wphys, t.Cp)[:, :, :, wp:wp + t.W]
    return b[:t.N * t.npos * t.row_stride].view(t.N, t.T, t.H, t.W, t.row_stride)


def ndhwc(t, clips):
    """The C valid channels of TRef t as [n, T, H, W, C] for the selected clips (a copy)."""
    return full_rows(t)[clips][..., t.ch_off:t.ch_off + t.C].clone()


def ncdhw64(t, clips):
    return ndhwc(t, clips).permute(0, 4, 1, 2, 3).double()


def rows64(t, clips):
    """[n, npos, C] float64 (token tensors and pooled rows)."""
    return ndhwc(t, clips).reshape(len(clips), t.npos, t.C).double()


def buf_view(b, shape):
    n = math.prod(shape)
    return b.tensor[:n].view(*shape)


def se_sums64(b, N, Cp, C, clips):
    """The int64 fixed-point (2^-24) per-(sample, channel) sums an SE accumulator holds, as float64."""
    return b.tensor[:2 * N * Cp].view(torch.int64).view(N, Cp)[clips, :C].double() * 2.0 ** -24


def _grid(rows, cls, thw):
    """[n, cls + THW, C] token rows -> the patch grid [n, C, T, H, W]."""
    n, _, C = rows.shape
    return rows[:, cls:].reshape(n, *thw, C).permute(0, 4, 1, 2, 3)


def _rows_of(grid):
    n, C = grid.shape[:2]
    return grid.permute(0, 2, 3, 4, 1).reshape(n, -1, C)


def _w16(w):
    """The f16 weights the kernel was packed with."""
    return w.detach().to(torch.float16).double()


# =====================================================================================================================
# per-kind: inputs (read before the op runs), output (after) and the comparison
# =====================================================================================================================
def gather_inputs(spec, clips):
    k = spec["kind"]
    dev = torch.device("cuda")
    if k == "to_ndhwc":
        return {"src": spec["src"][clips].clone()}
    if k == "conv":
        d = {"x": ncdhw64(spec["x"], clips)}
        d["res"] = ncdhw64(spec["residual"], clips) if spec["residual"] is not None else None
        if spec["addend"] is not None:
            a, off = spec["addend"]
            co = spec["weight"].shape[0]
            full = full_rows(a)[clips][..., a.ch_off + off:a.ch_off + off + co]
            d["addend"] = full.permute(0, 4, 1, 2, 3).double()
        return d
    if k == "tap_sum":
        return {"x": ndhwc(spec["x"], clips).double()}
    if k == "fused_block":
        return {"x": ncdhw64(spec["x"], clips)}
    if k in ("pool", "token_conv", "copy_cls", "pos_cls", "head_reduce", "layernorm"):
        return {"x": rows64(spec["x"], clips), "x_raw": ndhwc(spec["x"], clips)}
    if k == "se_gate":
        x = spec["x"]
        return {"sums": se_sums64(spec["sums"], x.N, x.Cp, x.C, clips)}
    if k == "scale_act":
        x = spec["x"]
        g = buf_view(spec["gate"], (x.N, x.Cp))[clips, :x.C].double() if spec["gate"] is not None else None
        return {"x": rows64(x, clips), "gate": g}
    if k == "add_layernorm":
        return {"a": rows64(spec["a"], clips).float(), "br": rows64(spec["br"], clips).float()}
    if k == "layernorm_sets":
        return {"x": rows64(spec["x"], clips), "y": rows64(spec["y"], clips)}
    if k == "attention":
        return {n: rows64(spec[n], clips) for n in ("q", "k", "v")}
    raise AssertionError("no reference for %s" % k)


def _heads(r, H):
    n, N, C = r.shape
    return r.view(n, N, H, C // H).permute(0, 2, 1, 3)


def compare(spec, inp, clips, launched, cpu_ref=False):
    """Run the comparison of one op; returns [(what, err / tol)] (0.0 for bit-exact checks).  cpu_ref: compute the
    float64 reference on the CPU instead (self-check of the GPU path) and return it instead of comparing."""
    k = spec["kind"]
    if cpu_ref is not False:
        inp = {n: (v.to(cpu_ref) if torch.is_tensor(v) else v) for n, v in inp.items()}
    n = len(clips)
    out = []

    def bound(got, ref, absref, K, acc_eps=TS.ACC_EPS, extra=None, rnd=TS.F16_EPS, what=k):
        if cpu_ref is not False:
            out.append((what, ref))
            return
        r = TS.assert_close_to_f64(got, ref, absref, K, acc_eps=acc_eps, what=what, extra64=extra, rnd_eps=rnd)
        out.append((what, r[0]))

    def exact(got, want, what=k):
        if cpu_ref is not False:
            out.append((what, want.double()))
            return
        g, w = got.contiguous(), want.to(got.dtype).contiguous()
        bits = {torch.float16: torch.int16, torch.float32: torch.int32}[g.dtype]
        diff = g.view(bits) != w.view(bits)
        assert not bool(diff.any()), "%s: %d elements differ from the bit-exact reference" % (what, int(diff.sum()))
        out.append((what, 0.0))

    if k == "to_ndhwc":
        y = spec["y"]
        exact(ndhwc(y, clips) if cpu_ref is False else None, inp["src"].permute(0, 2, 3, 4, 1).to(torch.float16))
    elif k == "conv":
        w = _w16(spec["weight"])
        x = inp["x"]
        ref, absref = TS.conv_ref64(x, w, spec["scale"], spec["bias"], spec["stride"], spec["padding"],
                                    spec["dilation"], spec["groups"], ACT_NAME[spec["act"]], inp["res"])
        if spec["addend"] is not None:
            ref, absref = ref + inp["addend"], absref + inp["addend"].abs()
        K = w.shape[1] * math.prod(w.shape[2:])
        got = ncdhw64(spec["y"], clips) if cpu_ref is False else None
        bound(got, ref, absref, K)
        if spec["se_sums"] is not None:
            y = spec["y"]
            ntaps = math.prod(w.shape[2:])
            ref_s, npos = ref.sum(dim=(2, 3, 4)), ref[0, 0].numel()
            if cpu_ref is not False:
                out.append(("se_sums", ref_s))
            else:
                # the SE-sum bound of test_depthwise_instance (fp32 sums of the pre-rounding outputs, fixed point)
                sums = se_sums64(spec["se_sums"], y.N, y.Cp, y.C, clips).cpu()
                ref_s, absref_s = ref_s.cpu(), absref.sum(dim=(2, 3, 4)).cpu()
                tol = 2.0 ** -20 * (1 + ntaps / 64.0) * absref_s + npos * 2.0 ** -23 + 2.0 ** -22 * ref_s.abs()
                if any(i.startswith(("dwconv3d_kernel<", "dwconv3d_w4_kernel<")) for i in launched):
                    tol = tol + TS.F16_EPS * ref.abs().sum(dim=(2, 3, 4)).cpu()
                r = float(((sums - ref_s).abs() / tol).max())
                assert r <= 1.0, "se_sums: err/tol %.3g" % r
                out.append(("se_sums", r))
    elif k == "tap_sum":
        x, y = inp["x"], spec["y"]
        co, kt, st, pt, dil = y.C, spec["kt"], spec["st"], spec["pt"], spec["dil"]
        cop = PK.pad8(co)
        Ti, To = x.shape[1], y.T
        acc = torch.zeros(n, To, y.H, y.W, co, dtype=torch.float64, device=x.device)
        aab = torch.zeros_like(acc)
        for t in range(To):
            for d in range(kt):
                ti = t * st + d * dil - pt
                if 0 <= ti < Ti:
                    tap = x[:, ti, :, :, d * cop:d * cop + co]
                    acc[:, t] += tap
                    aab[:, t] += tap.abs()
        sc, bi = spec["scale"].double().to(x.device), spec["bias"].double().to(x.device)
        pre = acc * sc + bi
        act = ACT_NAME[spec["act"]]
        absref = TS.LIP[act] * (aab * sc.abs() + bi.abs())
        got = ndhwc(y, clips) if cpu_ref is False else None
        bound(got, TS.act64(pre, act), absref, kt + 2, acc_eps=TS.SUM_EPS, extra=TS.act_err64(pre, act))
    elif k == "fused_block":
        wa, wb, wc = (_w16(spec[n]) for n in ("wa", "wb", "wc"))
        ws = _w16(spec["ws"]) if spec["ws"] is not None else None
        yr, _, _, Y, prop = TS.fused_block_ref64(inp["x"], wa, wb, wc, ws, spec["folds"], spec["kt"], spec["sb"],
                                                 ACT_NAME[spec["act"]])
        K = wa.shape[0] + (wa.shape[1] if ws is not None else 0)
        got = ncdhw64(spec["y"], clips) if cpu_ref is False else None
        bound(got, yr, Y, K, extra=prop)
    elif k == "pool":
        x, y, cls = spec["x"], spec["y"], spec["cls"]
        thw = spec.get("thw", (x.T, x.H, x.W))
        g = _grid(inp["x"], cls, thw)
        kk, s, p = spec["kernel"], spec["stride"], spec["padding"]
        pad = (p[2], p[2], p[1], p[1], p[0], p[0])
        got = rows64(y, clips)[:, cls:] if cpu_ref is False else None
        if spec["mode"] == L.POOL_MAX:
            ref = F.max_pool3d(F.pad(g, pad, value=-math.inf), kk, s)
            exact(got.to(torch.float16) if got is not None else None, _rows_of(ref).to(torch.float16))
        else:
            ref = F.avg_pool3d(F.pad(g, pad), kk, s)
            absref = F.avg_pool3d(F.pad(g.abs(), pad), kk, s)
            glob = "global_pool_kernel" in launched
            K = (math.ceil(math.prod(thw) / 32) + 32) if glob else math.prod(kk)
            bound(got, _rows_of(ref), _rows_of(absref), K, acc_eps=TS.SUM_EPS)
    elif k == "token_conv":
        x, y, cls = spec["x"], spec["y"], spec["cls"]
        g = _grid(inp["x"], cls, spec["thw"])
        w = _w16(spec["weight"])
        C = w.shape[0]
        ones = torch.ones(C, dtype=torch.float64)
        ref, absref = TS.conv_ref64(g, w, ones, torch.zeros_like(ones), spec["stride"], spec["padding"],
                                    spec["dilation"], C, "none", None)
        got = rows64(y, clips)[:, cls:] if cpu_ref is False else None
        bound(got, _rows_of(ref), _rows_of(absref), math.prod(w.shape[2:]))
    elif k == "copy_cls":
        exact(rows64(spec["y"], clips)[:, 0].to(spec["y"].buf.tensor.dtype) if cpu_ref is False else None,
              inp["x_raw"].reshape(n, -1, spec["x"].C)[:, 0])
    elif k == "pos_cls":
        y = spec["y"]
        xr = inp["x_raw"].reshape(n, -1, spec["x"].C).float()
        pos = spec["pos"].to(xr.device)
        hc = 1 if spec["has_cls"] else 0
        want = torch.empty(n, hc + xr.shape[1], xr.shape[2], dtype=torch.float32, device=xr.device)
        if hc:
            want[:, 0] = pos[0]
        want[:, hc:] = xr + pos[hc:]
        got = ndhwc(y, clips).reshape(n, y.npos, y.C) if cpu_ref is False else None
        exact(got, want.to(y.buf.tensor.dtype))
    elif k == "head_reduce":
        x64 = inp["x"]
        C = x64.shape[2]
        got = buf_view(spec["out"], (spec["x"].N, C))[clips] if cpu_ref is False else None
        if not spec["softmax"]:
            bound(got, x64.mean(1), x64.abs().mean(1), x64.shape[1] + 1, acc_eps=TS.SUM_EPS, rnd=TS.F32_EPS)
        else:
            p = torch.softmax(x64, 2)
            d = x64 - x64.max(2, keepdim=True).values
            rel = 2.0 ** -22 + TS.F32_EPS * d.abs()
            extra = (p * (rel + rel.max(2, keepdim=True).values)).mean(1)
            D = -(-C // 256) + 13
            bound(got, p.mean(1), p.mean(1), x64.shape[1] + D + 3, acc_eps=TS.SUM_EPS, extra=extra, rnd=TS.F32_EPS)
    elif k == "se_gate":
        x = spec["x"]
        dev = inp["sums"].device
        mean = inp["sums"] / x.npos
        w1, b1, w2, b2 = (spec[n].double().to(dev) for n in ("w1", "b1", "w2", "b2"))
        hid = (b1 + mean @ w1.t()).clamp_min(0)
        a = b2 + hid @ w2.t()
        gate = torch.sigmoid(a)
        Hm = b1.abs() + mean.abs() @ w1.abs().t()
        A = b2.abs() + Hm @ w2.abs().t()
        extra = gate * (1 - gate) * (2 + 1.173 * a.abs()) * 2.0 ** -23 + TS.F32_EPS * gate
        got = buf_view(spec["gate"], (x.N, x.Cp))[clips, :x.C] if cpu_ref is False else None
        bound(got, gate, 0.25 * A, x.C + w1.shape[0] + 3, acc_eps=TS.SUM_EPS, extra=extra, rnd=TS.F32_EPS)
    elif k == "scale_act":
        x = spec["x"]
        v = inp["x"]
        if inp["gate"] is not None:
            v = v * inp["gate"].unsqueeze(1)
        act = ACT_NAME[spec["act"]]
        got = rows64(spec["y"], clips) if cpu_ref is False else None
        bound(got, TS.act64(v, act), TS.LIP[act] * v.abs(), 0, acc_eps=TS.F32_EPS, extra=TS.act_err64(v, act))
    elif k == "layernorm":
        v = inp["x"][:, :1] if spec["first_row_only"] else inp["x"]
        C = v.shape[2]
        name = next(iter(launched))
        _, lpr, nch = TS.ln_dispatch(C) if name in ("layernorm_reg_kernel", "add_layernorm_kernel") else \
            ("layernorm_kernel", 32, -(-(-(-C // 8)) // 32))
        ref, absref, K, extra = TS.ln_ref64(v.reshape(-1, 1, C), spec["gamma"].view(1, -1), spec["beta"].view(1, -1), 1,
                                            nch * 8 + int(math.log2(lpr)), spec["eps"])
        got = rows64(spec["y"], clips).reshape(-1, 1, C) if cpu_ref is False else None
        bound(got, ref, absref, K, acc_eps=TS.SUM_EPS, extra=extra)
    elif k == "add_layernorm":
        s = inp["a"] + inp["br"]                               # fp32, as the kernel adds
        if spec["s"] is not None:
            exact(ndhwc(spec["s"], clips).reshape(s.shape) if cpu_ref is False else None, s, what="add_layernorm.sum")
        if spec["y"] is not None:
            C = s.shape[2]
            _, lpr, nch = TS.ln_dispatch(C)
            ref, absref, K, extra = TS.ln_ref64(s.reshape(-1, 1, C), spec["gamma"].view(1, -1),
                                                spec["beta"].view(1, -1), 1, nch * 8 + int(math.log2(lpr)), spec["eps"])
            got = rows64(spec["y"], clips).reshape(-1, 1, C) if cpu_ref is False else None
            bound(got, ref, absref, K, acc_eps=TS.SUM_EPS, extra=extra)
    elif k == "layernorm_sets":
        x, y, cls, hd = spec["x"], spec["y"], spec["cls"], spec["head_dim"]
        v = inp["y"].clone()
        if cls:
            v[:, 0] = inp["x"][:, 0]
        C = v.shape[2]
        G = C // hd
        nsets = spec["gamma"].numel() // hd
        name = next(iter(launched))
        _, lpr, nch = TS.ln_dispatch(hd) if name == "layernorm_reg_kernel" else \
            ("layernorm_kernel", 32, -(-(-(-hd // 8)) // 32))
        ref, absref, K, extra = TS.ln_ref64(v.reshape(-1, G, hd), spec["gamma"].view(nsets, hd),
                                            spec["beta"].view(nsets, hd), G // nsets, nch * 8 + int(math.log2(lpr)),
                                            spec["eps"])
        got = rows64(y, clips).reshape(-1, G, hd) if cpu_ref is False else None
        bound(got, ref, absref, K, acc_eps=TS.SUM_EPS, extra=extra)
    elif k == "attention":
        H = spec["heads"]
        q, kk, v = (_heads(inp[m], H) for m in ("q", "k", "v"))
        ref, absref = TS.attn_ref64(q, kk, v, spec["scale"], spec["residual"])
        back = lambda t: t.permute(0, 2, 1, 3).reshape(n, t.shape[2], -1)        # noqa: E731
        got = rows64(spec["o"], clips) if cpu_ref is False else None
        bound(got, back(ref), back(absref), 0, acc_eps=TS.ACC_EPS_ATTN)
    else:
        raise AssertionError("no reference for %s" % k)
    return out


def _outputs(spec):
    return [t for t in record_io(spec)[1] if isinstance(t, TRef)]


def check_layout(spec, before):
    """Pad channels of every TRef output are zero; channels of its rows outside [ch_off, ch_off + Cp) are as they were
    before the op (other producers' slices of a concat buffer)."""
    for i, t in enumerate(_outputs(spec)):
        rows = full_rows(t)
        pad = rows[..., t.ch_off + t.C:t.ch_off + t.Cp]
        assert not bool(pad.any()), "pad channels [%d, %d) not zero" % (t.C, t.Cp)
        if before[i] is not None:
            was = before[i]
            keep = torch.ones(t.row_stride, dtype=torch.bool, device=rows.device)
            keep[t.ch_off:t.ch_off + t.Cp] = False
            same = torch.equal(rows[..., keep], was[..., keep])
            assert same, "channels outside this op's slice of the shared buffer changed"


def build_workload(name, use_graph=False, batch=None):
    from pytorchvideo_b200.engine import compile_model
    model, B, T, H, W, is_sf = bench.build_model_and_inputs(name, batch)

    def inputs(seed):
        x = bench.make_inputs(B, T, H, W, is_sf, seed=seed)
        return [t.cuda() for t in (x if is_sf else [x])]
    ins, alt = inputs(42), inputs(43)           # bench.py's inputs, and a second set for the replay
    cm = compile_model(model, ins if is_sf else ins[0], dtype="f16", use_graph=use_graph)
    return cm, ins, alt, B


def stage(cm, ins):
    for s, t in zip(cm.static_in, ins):
        s.copy_(t)


def audit_plan(plan, clips, corrupt=None, cpu_check=None):
    """Walk the plan on one stream, comparing every op with its float64 reference.  Returns (failures, stats):
    failures [(op index, name, message)], stats {family: (launches, largest err / tol, instances)}.
    corrupt(i, spec): called after op i ran, before its comparison.  cpu_check: a dict filled with
    {kind: largest relative difference between the float64 references computed on the GPU and on the CPU} for the
    first op of each kind."""
    stream = torch.cuda.current_stream()
    sp = stream.cuda_stream
    failures, stats = [], {}
    for i, ((name, fn), spec) in enumerate(zip(plan.ops, plan.op_spec)):
        if spec is None:
            assert name.endswith(NO_VALUE_SUFFIXES), name
            fn(sp)
            continue
        try:
            inp = gather_inputs(spec, clips)
            before = [full_rows(t).clone() if (t.row_stride > t.Cp and t.padw is None) else None
                      for t in _outputs(spec)]
        except Exception as e:                          # noqa: BLE001 - reported with the op's name
            failures.append((i, name, "reading inputs: %r" % e))
            fn(sp)
            continue
        c0 = TS.kernel_counts()
        fn(sp)
        torch.cuda.synchronize()
        launched = TS.kernel_count_diff(c0, TS.kernel_counts())
        fam = family_of(spec)
        key = spec["route"] if spec["kind"] == "conv" else spec["kind"]
        if corrupt is not None:
            corrupt(i, spec)
        try:
            assert launched and all(n.startswith(fam) for n in launched), \
                "launched %s, outside the %s family" % (launched, key)
            res = compare(spec, inp, clips, launched)
            check_layout(spec, before)
        except AssertionError as e:
            failures.append((i, name, str(e)[:400]))
            continue
        if cpu_check is not None and spec["kind"] not in cpu_check:
            gpu = compare(spec, inp, clips, launched, cpu_ref=torch.device("cuda"))
            cpu = compare(spec, inp, clips, launched, cpu_ref=torch.device("cpu"))
            rel = 0.0
            for (_, g), (_, c) in zip(gpu, cpu):
                g, c = g.double().cpu(), c.double().cpu()
                rel = max(rel, float((g - c).abs().max()) / max(float(c.abs().max()), 1e-300))
            cpu_check[spec["kind"]] = rel
        n_, worst, inst = stats.get(key, (0, 0.0, set()))
        stats[key] = (n_ + 1, max([worst] + [r for _, r in res]), inst | set(launched))
    return failures, stats


def _bits(t):
    """Bit patterns: SE-sum buffers hold int64 fixed-point sums in f32 storage, some of which read as NaN."""
    return t.view({torch.float16: torch.int16, torch.float32: torch.int32}.get(t.dtype, t.dtype))


def _clips(B):
    return sorted({0, B // 2, B - 1})


# =====================================================================================================================
# GPU: the audit and the graph replay, per workload
# =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("name", WORKLOADS)
def test_workload_audit_and_graph_replay(name):
    t0 = time.time()
    cm, ins, alt, B = build_workload(name)
    plan = cm.plan
    stage(cm, ins)
    torch.cuda.synchronize()
    with torch.no_grad():
        failures, stats = audit_plan(plan, _clips(B))
    t_audit = time.time() - t0
    n_checked = sum(v[0] for v in stats.values())
    insts = set().union(*(v[2] for v in stats.values())) if stats else set()
    print("RESULT %s: %d launches, %d audited, %d instances, %.0f s; largest err/tol per family: %s" % (
        name, len(plan.ops), n_checked, len(insts), t_audit,
        ", ".join("%s %d x %.3f" % (k, v[0], v[1]) for k, v in sorted(stats.items()))))
    assert not failures, "\n".join("op %d %s: %s" % f for f in failures[:20])
    assert n_checked + sum(1 for s in plan.op_spec if s is None) == len(plan.ops)

    # ---- graph replay against the single-stream run, buffer for buffer
    single = [b.tensor.clone() for b in plan.bufs]
    for b in plan.bufs:
        b.tensor.zero_()
    cm._capture()
    for k, inputs in enumerate((ins, alt, ins)):
        stage(cm, inputs)
        cm.graph.replay()
        torch.cuda.synchronize()
        if k == 1:
            continue
        bad = [i for i, (b, s) in enumerate(zip(plan.bufs, single)) if not torch.equal(_bits(b.tensor), _bits(s))]
        assert not bad, "replay %d: %d of %d buffers differ from the single-stream run (first: buffer %d)" % (
            k, len(bad), len(single), bad[0])
    print("RESULT %s: graph replay (%d lanes) equals the single-stream run in all %d buffers, %.0f s in all" % (
        name, len(plan.sched["lanes"]), len(single), time.time() - t0))
    del single, cm, plan
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_audit_rejects_a_corrupted_tile_and_its_references_agree_with_the_cpu():
    """Self-checks on x3d_xs: one 128-row tile of one convolution output moved by 8 f16 ulp after its launch fails
    the audit under that op's name; and the float64 reference of the first op of each kind agrees between the GPU
    and the CPU to 1e-12 relative, whatever algorithm cuDNN picks on the GPU."""
    cm, ins, _, B = build_workload("x3d_xs")
    plan = cm.plan
    target = next(i for i, s in enumerate(plan.op_spec) if s is not None and s["kind"] == "conv"
                  and s["route"] == "tcgen05" and s["y"].N * s["y"].npos >= 4 * 128 and i > 2)

    def corrupt(i, spec):
        if i == target:
            y = spec["y"]
            rows = full_rows(y).reshape(-1, y.row_stride)
            tile = rows[128:256, y.ch_off:y.ch_off + y.C]
            tile.view(torch.int16).add_(8)
    stage(cm, ins)
    cpu_check = {}
    with torch.no_grad():
        failures, _ = audit_plan(plan, [0], corrupt=corrupt, cpu_check=cpu_check)
    names = [f[1] for f in failures]
    assert names == [plan.ops[target][0]], failures
    print("RESULT self-check: corrupted %s rejected (%s); GPU vs CPU float64 references: %s" % (
        names[0], failures[0][2][:120], cpu_check))
    assert cpu_check and all(r <= 1e-12 for r in cpu_check.values()), cpu_check


# =====================================================================================================================
# CPU: records, declared I/O, module agreement
# =====================================================================================================================
_PLANS = {}


def _lowered(name):
    if name not in _PLANS:
        from pytorchvideo_b200.engine.lower import lower_only
        model, B, T, H, W, is_sf = bench.build_model_and_inputs(name)
        shape = (B, 3, T, H, W)
        x = torch.empty(shape)
        plan, _ = lower_only(model, TS.slowfast_inputs(x) if is_sf else x)
        _PLANS.clear()
        _PLANS[name] = (plan, model)
    return _PLANS[name]


EXPECTED_LAUNCHES = {"slowfast_r50": 103, "x3d_m": 135, "x3d_xs": 135, "slow_r50": 58, "csn_r101": 109,
                     "r2plus1d_r50": 73, "mvit_base_16x4": 165}


@pytest.mark.parametrize("name", WORKLOADS)
def test_every_launch_has_a_checked_record(name):
    plan, _ = _lowered(name)
    assert len(plan.op_spec) == len(plan.ops) == EXPECTED_LAUNCHES[name]
    missing = [n for (n, _), s in zip(plan.ops, plan.op_spec) if not supported(s) and not n.endswith(NO_VALUE_SUFFIXES)]
    assert not missing, missing
    for (n, _), s in zip(plan.ops, plan.op_spec):
        if s is None:
            continue
        for t in record_io(s)[0] + record_io(s)[1]:
            assert isinstance(t, (TRef, Buf)), (n, t)


def _io_problems(plan):
    bad = []
    for (n, _), s, io in zip(plan.ops, plan.op_spec, plan.op_io):
        if io is None or s is None:
            continue
        ins, outs = record_io(s)
        if not _bufs(ins) <= _bufs(io[0]):
            bad.append((n, "reads"))
        if not _bufs(outs) <= _bufs(io[1]):
            bad.append((n, "writes"))
    return bad


@pytest.mark.parametrize("name", WORKLOADS)
def test_declared_io_covers_the_records(name):
    plan, _ = _lowered(name)
    assert not _io_problems(plan)


@pytest.mark.parametrize("case", sorted(c for c, v in TS.AUDIO_CASES.items() if v[2][0] == "avsf"))
def test_declared_io_covers_the_records_audio(case):
    """AVSlowFast lanes read across pathways: a missing declaration would be a cross-lane race."""
    from pytorchvideo_b200.engine.lower import lower_only
    from pytorchvideo_b200 import models as M
    m, x = TS.build_audio_case(case, M, seed=2024)
    plan, _ = lower_only(m, x)
    assert len(set(plan.op_lane)) > 1
    assert not _io_problems(plan)


_ACT_OF = {"ReLU": L.ACT_RELU, "SiLU": L.ACT_SWISH, "Swish": L.ACT_SWISH, "GELU": L.ACT_GELU}


@pytest.mark.parametrize("name", WORKLOADS)
def test_records_agree_with_their_modules(name):
    plan, model = _lowered(name)
    mods = dict(model.named_modules())
    checked = 0
    for (n, _), s in zip(plan.ops, plan.op_spec):
        m = mods.get(n)
        if s is None or s["kind"] != "conv" or type(m).__name__ != "Conv3d":
            continue
        assert s["stride"] == tuple(m.stride) and s["padding"] == tuple(m.padding), n
        assert s["dilation"] == tuple(m.dilation), n
        # grouped convolutions the library does not take run as dense block-diagonal convolutions
        assert s["groups"] == m.groups or (s["groups"] == 1 and s["weight"].shape[1] == m.in_channels), n
        assert tuple(s["weight"].shape[0:1]) == (m.out_channels,) and s["x"].C == m.in_channels, n
        parent, _, leaf = n.rpartition(".")
        # conv_a's activation is fused into it in every family (conv_b's may follow an SE block instead)
        act = getattr(mods.get(parent), "act_a", None) if leaf == "conv_a" else None
        if act is not None and type(act).__name__ in _ACT_OF:
            assert s["act"] == _ACT_OF[type(act).__name__], n
        checked += 1
    for (n, _), s in zip(plan.ops, plan.op_spec):
        m = mods.get(n)
        if s is not None and s["kind"] == "conv" and type(m).__name__ == "Linear":
            assert tuple(s["weight"].shape) == (m.out_features, m.in_features, 1, 1, 1), n
            assert (s["stride"], s["padding"], s["groups"]) == ((1, 1, 1), (0, 0, 0), 1), n
            checked += 1
        if s is not None and s["kind"] in ("token_conv", "pool") and s.get("modules"):
            t3 = lambda v: tuple(v) if isinstance(v, (tuple, list)) else (v,) * 3       # noqa: E731
            for m in s["modules"]:                      # pool_k and pool_v of a fused K | V pool
                assert t3(m.stride) == tuple(s["stride"]) and t3(m.padding) == tuple(s["padding"]), n
                assert t3(m.kernel_size) == tuple(s["weight"].shape[2:] if s["kind"] == "token_conv" else s["kernel"]), n
            checked += 1
        if s is not None and s["kind"] == "fused_block":
            for mod, w in zip(s["modules"], (s["wa"], s["wb"], s["wc"], s["ws"])):
                assert (mod is None and w is None) or mod.weight is w, n
            ca, cb = s["modules"][:2]
            assert s["kt"] == ca.kernel_size[0] and s["sb"] == cb.stride[1], n
            checked += 1
    assert checked >= 10, checked
