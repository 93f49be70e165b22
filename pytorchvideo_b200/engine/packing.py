"""Host-side, one-off parameter preparation: BatchNorm folding and weight re-layout.

This is set-up work done once per compiled plan (the analogue of the reference's
``EfficientBlockBase.convert`` step, accelerator/efficient_blocks/efficient_block_base.py:8-35 and
layers/accelerator/mobile_cpu/convolutions.py:120-175 where BN is fused at convert time); it is
not on the per-clip hot path.
"""
import torch


def pad8(c):
    return (int(c) + 7) // 8 * 8


def pad_to(c, m):
    return (int(c) + m - 1) // m * m


def fold_bn(conv_bias, bn, c_out, c_out_pad):
    """Return (scale, bias) fp32 CPU tensors of length c_out_pad for y = conv*scale + bias.

    Eval-mode BatchNorm: y = (x - mean) / sqrt(var + eps) * gamma + beta, folded over an optional
    convolution bias.  Pad lanes get scale = bias = 0 so padded channels stay exactly zero.
    """
    scale = torch.ones(c_out, dtype=torch.float64)
    bias = torch.zeros(c_out, dtype=torch.float64)
    if conv_bias is not None:
        bias = conv_bias.detach().double().cpu().clone()
    if bn is not None:
        var = bn.running_var.detach().double().cpu()
        mean = bn.running_mean.detach().double().cpu()
        gamma = bn.weight.detach().double().cpu() if bn.weight is not None else torch.ones(c_out, dtype=torch.float64)
        beta = bn.bias.detach().double().cpu() if bn.bias is not None else torch.zeros(c_out, dtype=torch.float64)
        s = gamma / torch.sqrt(var + bn.eps)
        bias = (bias - mean) * s + beta
        scale = s
    out_s = torch.zeros(c_out_pad, dtype=torch.float32)
    out_b = torch.zeros(c_out_pad, dtype=torch.float32)
    out_s[:c_out] = scale.float()
    out_b[:c_out] = bias.float()
    # where the vectors come from, for the in-place weight refresh of a compiled plan (engine/refresh.py)
    out_s._pv_fold, out_b._pv_fold = (conv_bias, bn, int(c_out), 0), (conv_bias, bn, int(c_out), 1)
    return out_s, out_b


def pack_dense_direct(w, ci_pad, co_pad, dtype):
    """[Co, Ci, kt, kh, kw] -> [taps, ci_pad, co_pad] (co contiguous)."""
    co, ci, kt, kh, kw = w.shape
    out = torch.zeros(kt * kh * kw, ci_pad, co_pad, dtype=dtype)
    out[:, :ci, :co] = w.detach().cpu().permute(2, 3, 4, 1, 0).reshape(kt * kh * kw, ci, co).to(dtype)
    return out.contiguous()


def pack_depthwise(w, c_pad, dtype):
    """[C, 1, kt, kh, kw] -> [taps, c_pad]."""
    c, one, kt, kh, kw = w.shape
    assert one == 1
    out = torch.zeros(kt * kh * kw, c_pad, dtype=dtype)
    out[:, :c] = w.detach().cpu().reshape(c, kt * kh * kw).t().to(dtype)
    return out.contiguous()


def pack_dense_tcgen05(w, ci_pad64, co_pad):
    """[Co, Ci, kt, kh, kw] -> [co_pad, pad64(taps * ci_pad64)] f16, K-major (k = tap * ci_pad64 + ci).

    TMA-fed kernel: ci_pad64 is a multiple of 64.  Gather-fed kernel (C_in < 64): ci_pad64 is the
    padded channel count itself and only the row end is padded to a multiple of 64."""
    co, ci, kt, kh, kw = w.shape
    taps = kt * kh * kw
    out = torch.zeros(co_pad, taps, ci_pad64, dtype=torch.float16)
    out[:co, :, :ci] = w.detach().cpu().permute(0, 2, 3, 4, 1).reshape(co, taps, ci).to(torch.float16)
    out = out.reshape(co_pad, taps * ci_pad64)
    k = out.shape[1]
    kp = pad_to(k, 64)
    if kp != k:
        out = torch.cat([out, torch.zeros(co_pad, kp - k, dtype=torch.float16)], 1)
    return out.contiguous()


def pack_grouped_tcgen05(w, groups, span_groups, span_k):
    """Grouped mode of the TMA-fed kernel: [Co, Cg_in, kt, kh, kw] -> f16 [Co, taps * span_k], K-major
    (k = tap * span_k + c).  Output channel co belongs to group g = co // Cg_out, which sits at input offset
    (g % span_groups) * Cg_in of its span; the rest of the row is zero (a block-diagonal GEMM per span)."""
    co, cgi, kt, kh, kw = w.shape
    cgo = co // groups
    taps = kt * kh * kw
    out = torch.zeros(co, taps, span_k, dtype=torch.float16)
    src = w.detach().cpu().permute(0, 2, 3, 4, 1).reshape(co, taps, cgi).to(torch.float16)
    for g in range(groups):
        off = (g % span_groups) * cgi
        out[g * cgo:(g + 1) * cgo, :, off:off + cgi] = src[g * cgo:(g + 1) * cgo]
    return out.reshape(co, taps * span_k).contiguous()


def expand_grouped_dense(w, groups):
    """[Co, Cg_in, kt, kh, kw] -> the block-diagonal dense weight [Co, groups * Cg_in, kt, kh, kw] (same dtype): a
    grouped convolution as an ordinary one, for the shapes the grouped mode does not take."""
    co, cgi = w.shape[:2]
    cgo = co // groups
    src = w.detach().cpu()
    out = torch.zeros((co, groups * cgi) + tuple(w.shape[2:]), dtype=src.dtype)
    for g in range(groups):
        out[g * cgo:(g + 1) * cgo, g * cgi:(g + 1) * cgi] = src[g * cgo:(g + 1) * cgo]
    return out


def window_lead(w_pad, pw, ci_pad):
    """Leading zero pixels of the window so that its first byte is 16-byte aligned (see pv_igemm.cu)."""
    return 1 if ((w_pad - pw) * ci_pad * 2) % 16 else 0


def window_elems(kw, ci_pad, lead=0):
    run = (kw + lead) * ci_pad
    return 16 if run <= 16 else (32 if run <= 32 else 64)


def pack_dense_window(w, ci_pad, co_pad, lead=0):
    """Window-mode stems: [Co, Ci, kt, kh, kw] -> [co_pad, kt*kh*win] f16 with
    k = (dt*kh+dh)*win + (lead+dw)*ci_pad + c  (win = 16|32|64; leading / trailing window elements
    multiply neighbouring-pixel data by zero)."""
    co, ci, kt, kh, kw = w.shape
    win = window_elems(kw, ci_pad, lead)
    out = torch.zeros(co_pad, kt * kh, win, dtype=torch.float16)
    src = w.detach().cpu().permute(0, 2, 3, 4, 1).reshape(co, kt * kh, kw, ci).to(torch.float16)
    tmp = torch.zeros(co, kt * kh, kw, ci_pad, dtype=torch.float16)
    tmp[..., :ci] = src
    out[:co, :, lead * ci_pad: (lead + kw) * ci_pad] = tmp.reshape(co, kt * kh, kw * ci_pad)
    return out.reshape(co_pad, kt * kh * win).contiguous()


def pack_rows_k16(w, ci_pad, co_pad):
    """[Co, Ci, kt, kh, kw] -> f16 [co_pad][pad16(taps * ci_pad)], k = tap * ci_pad + ci (zero padded): the
    [n][k] operand layout of the fused bottleneck kernel (csrc/pv_fastblock.cu)."""
    co, ci, kt, kh, kw = w.shape
    taps = kt * kh * kw
    k = taps * ci_pad
    kp = (k + 15) // 16 * 16
    out = torch.zeros(co_pad, kp, dtype=torch.float16)
    t = torch.zeros(co, taps, ci_pad, dtype=torch.float16)
    t[:, :, :ci] = w.detach().cpu().permute(0, 2, 3, 4, 1).reshape(co, taps, ci).to(torch.float16)
    out[:co, :k] = t.reshape(co, k)
    return out.contiguous()


def pack_stem_rows(w, ci_pad, co_pad, lead=0):
    """Stem-rows kernel (csrc/pv_stem.cu): the window packing of ``pack_dense_window`` re-ordered to the canonical
    no-swizzle K-major wgmma layout with all output channels of a 16-byte K chunk contiguous:
    [Co, Ci, kt, kh, kw] -> f16 [K / 8][pad16(co_pad)][8]."""
    rows = pack_dense_window(w, ci_pad, co_pad, lead)            # [co_pad, K]
    n16 = (co_pad + 15) // 16 * 16
    k = rows.shape[1]
    full = torch.zeros(n16, k, dtype=torch.float16)
    full[:co_pad] = rows
    return full.reshape(n16, k // 8, 8).permute(1, 0, 2).contiguous()


def pack_stem_stream(w, ci_pad, co_pad, lead=0):
    """Temporal-streaming stem (csrc/pv_stem_stream.cu): [Co, Ci, kt, kh, kw] -> f16 [K / 8][kt * co_pad][8] with
    K = kh * win.  The layout of ``pack_stem_rows`` for the (1, kh, kw) filter of every temporal tap side by side:
    column j * co_pad + c holds tap j of output channel c (no padding of the kt * co_pad columns to 16)."""
    co, ci, kt, kh, kw = w.shape
    n = kt * co_pad
    taps = torch.zeros(n, ci, 1, kh, kw, dtype=w.dtype)
    src = w.detach().cpu()
    for j in range(kt):
        taps[j * co_pad: j * co_pad + co] = src[:, :, j:j + 1]
    rows = pack_dense_window(taps, ci_pad, n, lead)               # [n, K]
    k = rows.shape[1]
    return rows.reshape(n, k // 8, 8).permute(1, 0, 2).contiguous()
