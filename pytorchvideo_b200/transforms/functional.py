"""Clip transforms executed by ONE fused CUDA kernel (pv_clip_transform_fwd).

Host side only computes small integer/weight tables (temporal indices, bilinear taps, crop
window) exactly as the reference's host code does; every pixel is touched on the GPU once.
Reference: transforms/functional.py:19-41, 92-160, 302-347, 604-615; transforms/transforms.py.
"""
import ctypes as C
import math

import numpy as np
import torch

from .. import _lib as L
from .mix import convert_to_one_hot  # noqa: F401

_DT = {torch.uint8: L.PV_U8, torch.float32: L.PV_F32, torch.float16: L.PV_F16}
_TABLE_CACHE = {}


def temporal_indices(t, num_samples):
    """clamp(torch.linspace(0, t-1, n), 0, t-1).long() - literally the reference's host
    expression (functional.py:39-40), so indices are bit-identical to the reference's."""
    assert num_samples > 0 and t > 0
    idx = torch.clamp(torch.linspace(0, t - 1, num_samples), 0, t - 1).long()
    return idx


def short_side_size(h, w, size):
    if w < h:
        return int(math.floor((float(h) / w) * size)), size
    return size, int(math.floor((float(w) / h) * size))


def bilinear_table(in_size, out_size):
    """(i0, i1, lambda1) of ATen's upsample_bilinear2d(align_corners=False) in fp32."""
    if in_size == out_size:
        i = np.arange(out_size, dtype=np.int32)
        return i, i.copy(), np.zeros(out_size, np.float32)
    scale = np.float32(in_size) / np.float32(out_size)
    d = np.arange(out_size, dtype=np.float32) + np.float32(0.5)
    # fma(scale, d, -0.5) with one rounding; astype, not np.float64(d), which turns a one-element array (out_size 1)
    # into a scalar
    src = (np.float64(scale) * d.astype(np.float64) - 0.5).astype(np.float32)
    src = np.maximum(src, np.float32(0))
    i0 = np.minimum(np.floor(src).astype(np.int64), in_size - 1)
    l1 = np.clip(src - i0.astype(np.float32), np.float32(0), np.float32(1)).astype(np.float32)
    i1 = i0 + (i0 < in_size - 1)
    return i0.astype(np.int32), i1.astype(np.int32), l1


def center_crop_window(h, w, size):
    th, tw = (size, size) if isinstance(size, int) else size
    if th > h or tw > w:
        raise ValueError("crop size %s larger than image (%d, %d)" % ((th, tw), h, w))
    return int(round((h - th) / 2.0)), int(round((w - tw) / 2.0)), th, tw


def uniform_crop_window(h, w, size, spatial_idx):
    assert spatial_idx in (0, 1, 2)
    y = int(math.ceil((h - size) / 2))
    x = int(math.ceil((w - size) / 2))
    if h > w:
        y = 0 if spatial_idx == 0 else (h - size if spatial_idx == 2 else y)
    else:
        x = 0 if spatial_idx == 0 else (w - size if spatial_idx == 2 else x)
    return y, x, size, size


def random_crop_window(h, w, size):
    """torchvision RandomCrop.get_params: offsets drawn on the host from torch's global RNG."""
    th, tw = (size, size) if isinstance(size, int) else size
    if h < th or w < tw:
        raise ValueError("Required crop size %s is larger than input image size %s" % ((th, tw), (h, w)))
    if w == tw and h == th:
        return 0, 0, h, w
    i = torch.randint(0, h - th + 1, size=(1,)).item()
    j = torch.randint(0, w - tw + 1, size=(1,)).item()
    return i, j, th, tw


def clip_transform(x, frame_idx=None, resize_hw=None, window=None, mean=None, std=None, div255=False,
                   out_dtype=torch.float32, out=None, hflip=False):
    """Run the fused kernel on a CUDA clip ``x`` of logical shape (C, T, H, W) (any strides).

    frame_idx : int tensor/sequence of frames to keep (None = all)
    resize_hw : (new_h, new_w) bilinear target (None = no resize)
    window    : (top, left, h, w) crop in the resized frame (None = full)
    mean/std  : per-channel normalisation (None = skip)
    hflip     : mirror the (cropped) output along W - torchvision hflip fused for free by reversing the
                column tap tables on the host
    """
    if not torch.is_tensor(x) or x.dim() != 4:
        raise RuntimeError("expected a (C, T, H, W) tensor")
    if x.device.type != "cuda":
        raise RuntimeError("pytorchvideo_b200 transforms run on the GPU only (no CPU path)")
    if x.dtype not in _DT:
        raise RuntimeError("unsupported clip dtype %s" % x.dtype)
    lib = L.load()
    Cc, T, H, W = x.shape
    idx = torch.arange(T) if frame_idx is None else torch.as_tensor(frame_idx).long().cpu()
    if idx.numel() == 0 or int(idx.min()) < 0 or int(idx.max()) >= T:
        raise RuntimeError("frame index out of range")
    nh, nw = (H, W) if resize_hw is None else resize_hw
    top, left, oh, ow = (0, 0, nh, nw) if window is None else window
    if top < 0 or left < 0 or top + oh > nh or left + ow > nw:
        raise RuntimeError("crop window outside the frame")
    y0, y1, ly = bilinear_table(H, nh)
    x0, x1, lx = bilinear_table(W, nw)
    y0, y1, ly = y0[top:top + oh], y1[top:top + oh], ly[top:top + oh]
    x0, x1, lx = x0[left:left + ow], x1[left:left + ow], lx[left:left + ow]
    if hflip:
        x0, x1, lx = x0[::-1], x1[::-1], lx[::-1]
    per_channel = mean is not None or std is not None
    n_t = int(idx.numel())
    if per_channel:
        if Cc > 4:
            raise RuntimeError("per-channel normalisation supports at most 4 channels")
        mean_l = [float(m) for m in (mean if mean is not None else [0.0] * Cc)]
        std_l = [float(s) for s in (std if std is not None else [1.0] * Cc)]
        if len(mean_l) == 1:
            mean_l = mean_l * Cc
        if len(std_l) == 1:
            std_l = std_l * Cc
        kC, kidx, ksc = Cc, idx, x.stride(0)
    else:
        # no per-channel state: fold channels into the frame list so any C works
        mean_l, std_l = [0.0], [1.0]
        kC = 1
        kidx = (torch.arange(Cc).view(-1, 1) * 0 + idx.view(1, -1)).reshape(-1)
        # address = c*stride_c + t*stride_t is not expressible with one stride unless we bake the
        # channel offset into the frame index; do it when stride_c is a multiple of stride_t,
        # otherwise run channel by channel.
        ksc = 0
        if Cc > 1:
            st_c, st_t = x.stride(0), x.stride(1)
            if st_t != 0 and st_c % st_t == 0:
                kidx = (torch.arange(Cc).view(-1, 1) * (st_c // st_t) + idx.view(1, -1)).reshape(-1)
            else:
                outs = [clip_transform(x[c:c + 1], frame_idx, resize_hw, window, None, None, div255, out_dtype)
                        for c in range(Cc)]
                return torch.cat(outs, 0)
    dev = x.device
    # device-side tables are tiny but cost several H2D copies: cache them per (geometry, device)
    ckey = (dev.index, H, W, nh, nw, top, left, oh, ow, bool(hflip), tuple(int(i) for i in kidx.tolist()))
    cached = _TABLE_CACHE.get(ckey)
    if cached is None:
        tabs = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (y0, y1, ly, x0, x1, lx)]
        idx_d = kidx.to(torch.int32).to(dev)
        if len(_TABLE_CACHE) > 256:
            _TABLE_CACHE.clear()
        _TABLE_CACHE[ckey] = (tabs, idx_d)
    else:
        tabs, idx_d = cached
    if out is None:
        out = torch.empty((Cc, n_t, oh, ow), dtype=out_dtype, device=dev)
    else:
        assert out.shape == (Cc, n_t, oh, ow) and out.is_contiguous() and out.dtype == out_dtype
    d = L.ClipTransformDesc()
    d.C, d.n_t, d.out_h, d.out_w = kC, int(idx_d.numel()), oh, ow
    d.sc, d.st, d.sh, d.sw = ksc, x.stride(1), x.stride(2), x.stride(3)
    for i in range(4):
        d.mean[i] = mean_l[i] if i < len(mean_l) else 0.0
        d.stdv[i] = std_l[i] if i < len(std_l) else 1.0
    d.src_dtype = _DT[x.dtype]
    d.dst_dtype = L.PV_F16 if out_dtype == torch.float16 else L.PV_F32
    d.div255 = 1 if div255 else 0
    stream = torch.cuda.current_stream(dev).cuda_stream
    L.check(lib.pv_clip_transform_fwd(C.byref(d), x.data_ptr(), idx_d.data_ptr(), tabs[0].data_ptr(),
                                      tabs[1].data_ptr(), tabs[2].data_ptr(), tabs[3].data_ptr(),
                                      tabs[4].data_ptr(), tabs[5].data_ptr(), out.data_ptr(), stream),
            "pv_clip_transform_fwd")
    # tables must outlive the asynchronous launch
    out._pv_keepalive = (tabs, idx_d)
    return out


_IDX_CACHE = {}


def _dev_i32(values, dev):
    key = (dev.index, tuple(int(v) for v in values))
    t = _IDX_CACHE.get(key)
    if t is None:
        if len(_IDX_CACHE) > 512:
            _IDX_CACHE.clear()
        t = _IDX_CACHE[key] = torch.tensor(list(key[1]), dtype=torch.int32, device=dev)
    return t


def slow_pathway_indices(n_frames, alpha):
    """SlowFastPackPathway (pytorchvideo_trainer/datamodule/transforms.py:129-136):
    torch.linspace(0, T - 1, T // alpha).long() - positions inside the (already subsampled) fast clip."""
    return torch.linspace(0, n_frames - 1, n_frames // alpha).long()


def _set_arith(d, Cc, mean, std, div255):
    """The /255 and normalisation fields of a ClipBatchDesc; one mean / std value stands for every channel."""
    normalize = mean is not None or std is not None
    mean_l = [float(m) for m in (mean if mean is not None else [0.0] * Cc)]
    std_l = [float(v) for v in (std if std is not None else [1.0] * Cc)]
    mean_l = mean_l * Cc if len(mean_l) == 1 else mean_l
    std_l = std_l * Cc if len(std_l) == 1 else std_l
    for i in range(4):
        d.mean[i] = mean_l[i] if i < len(mean_l) else 0.0
        d.stdv[i] = std_l[i] if i < len(std_l) else 1.0
    d.div255, d.normalize = 1 if div255 else 0, 1 if normalize else 0


def _slow_table(n_t, slow_alpha, dev):
    """(device slot of each kept frame in the slow pathway or -1, slow frame count)."""
    sidx = slow_pathway_indices(n_t, int(slow_alpha)).tolist()
    n_slow = len(sidx)
    if n_slow < 1:
        raise RuntimeError("slow pathway would be empty (n_t=%d, alpha=%d)" % (n_t, slow_alpha))
    pos = [-1] * n_t
    for k, j in enumerate(sidx):
        pos[j] = k           # linspace().long() is strictly increasing for alpha >= 1: every slot is unique
    if len(set(sidx)) != n_slow:
        raise RuntimeError("slow pathway indices repeat (alpha < 1?)")
    return _dev_i32(pos, dev), n_slow


def clip_transform_batch(x, frame_idx=None, resize_hw=None, window=None, mean=None, std=None, div255=False,
                         out_dtype=torch.float16, hflip=False, geom=None, slow_alpha=None, out=None, out_slow=None):
    """The fused chain on a BATCH of clips in one launch (pv_clip_transform_batch; taps computed in the kernel).

    x         : (B, C, T, H, W) CUDA tensor, C <= 4, any strides (CTHW-contiguous or the decoder's THWC-interleaved
                frames); a 4-D clip is a batch of one
    geom      : optional per-clip list of (resize_hw, window, hflip[, first_frame]) - the train chain with its own
                random short side / crop / flip per clip, or the spatial x temporal test-time views of one video
                (expand the video to a batch with clip stride 0); resize_hw / window then only give the output size
    slow_alpha: also emit the SlowFast slow pathway (frames linspace(0, n_t-1, n_t//alpha).long() of the kept
                frames) from the same pass; returns [slow, fast] like SlowFastPackPathway
    out_dtype : torch.float16 | torch.float32, or torch.uint8 for a pure frame selection / crop of uint8 clips
    """
    squeeze = False
    if torch.is_tensor(x) and x.dim() == 4:
        x, squeeze = x.unsqueeze(0), True
        out = out.unsqueeze(0) if out is not None and out.dim() == 4 else out
        out_slow = out_slow.unsqueeze(0) if out_slow is not None and out_slow.dim() == 4 else out_slow
    if not torch.is_tensor(x) or x.dim() != 5:
        raise RuntimeError("expected a (B, C, T, H, W) or (C, T, H, W) tensor")
    if x.device.type != "cuda":
        raise RuntimeError("pytorchvideo_b200 transforms run on the GPU only (no CPU path)")
    if x.dtype not in _DT:
        raise RuntimeError("unsupported clip dtype %s" % x.dtype)
    B, Cc, T, H, W = x.shape
    if Cc > 4:
        raise RuntimeError("at most 4 channels per clip (got %d)" % Cc)
    lib = L.load()
    dev = x.device
    idx = torch.arange(T) if frame_idx is None else torch.as_tensor(frame_idx).long().cpu()
    if idx.numel() == 0 or int(idx.min()) < 0 or int(idx.max()) >= T:
        raise RuntimeError("frame index out of range")
    n_t = int(idx.numel())
    nh, nw = (H, W) if resize_hw is None else (int(resize_hw[0]), int(resize_hw[1]))
    top, left, oh, ow = (0, 0, nh, nw) if window is None else (int(v) for v in window)
    geom_d = None
    if geom is not None:
        if len(geom) != B:
            raise RuntimeError("geom needs one entry per clip")
        flat = []
        for entry in geom:
            ghw, gwin, gflip = entry[:3]
            goff = int(entry[3]) if len(entry) > 3 else 0
            if goff + int(idx.min()) < 0 or goff + int(idx.max()) >= T:
                raise RuntimeError("view frame range outside the clip")
            gh, gw = (H, W) if ghw is None else ghw
            gt, gl, goh, gow = (0, 0, gh, gw) if gwin is None else gwin
            if (goh, gow) != (oh, ow) or gt < 0 or gl < 0 or gt + goh > gh or gl + gow > gw:
                raise RuntimeError("per-clip crop windows must have the common output size and lie inside the resized frame")
            flat += [int(gh), int(gw), int(gt), int(gl), 1 if gflip else 0, goff]
        geom_d = torch.tensor(flat, dtype=torch.int32, device=dev)
    elif top < 0 or left < 0 or top + oh > nh or left + ow > nw:
        raise RuntimeError("crop window outside the frame")
    d = L.ClipBatchDesc()
    d.C, d.n_clips, d.n_t = Cc, B, n_t
    d.in_h, d.in_w, d.new_h, d.new_w = H, W, nh, nw
    d.top, d.left, d.out_h, d.out_w, d.hflip = top, left, oh, ow, 1 if hflip else 0
    d.s_clip, d.sc, d.st, d.sh, d.sw = x.stride(0), x.stride(1), x.stride(2), x.stride(3), x.stride(4)
    _set_arith(d, Cc, mean, std, div255)
    d.src_dtype = _DT[x.dtype]
    if out_dtype not in _DT:
        raise RuntimeError("unsupported output dtype %s" % out_dtype)
    d.dst_dtype = _DT[out_dtype]
    if out is None:
        out = torch.empty((B, Cc, n_t, oh, ow), dtype=out_dtype, device=dev)
    elif tuple(out.shape) != (B, Cc, n_t, oh, ow) or not out.is_contiguous() or out.dtype != out_dtype:
        raise RuntimeError("out must be a contiguous %s tensor of shape %s" % (out_dtype, (B, Cc, n_t, oh, ow)))
    d.d_clip = out.stride(0)
    idx_d = _dev_i32(idx.tolist(), dev)
    slow_d, n_slow = None, 0
    if slow_alpha is not None:
        slow_d, n_slow = _slow_table(n_t, slow_alpha, dev)
        if out_slow is None:
            out_slow = torch.empty((B, Cc, n_slow, oh, ow), dtype=out_dtype, device=dev)
        elif tuple(out_slow.shape) != (B, Cc, n_slow, oh, ow) or not out_slow.is_contiguous() or out_slow.dtype != out_dtype:
            raise RuntimeError("out_slow has the wrong shape / dtype")
        d.n_slow, d.d_slow_clip = n_slow, out_slow.stride(0)
    stream = torch.cuda.current_stream(dev).cuda_stream
    L.check(lib.pv_clip_transform_batch(C.byref(d), x.data_ptr(), idx_d.data_ptr(),
                                        slow_d.data_ptr() if slow_d is not None else None,
                                        geom_d.data_ptr() if geom_d is not None else None, out.data_ptr(),
                                        out_slow.data_ptr() if out_slow is not None else None, stream),
            "pv_clip_transform_batch")
    out._pv_keepalive = (idx_d, slow_d, geom_d)     # device tables must outlive the asynchronous launch
    if squeeze:
        out = out[0]
        out_slow = out_slow[0] if out_slow is not None else None
    return [out_slow, out] if slow_alpha is not None else out


def ragged_tables(frame_off, geom, out_hw):
    """Host checks and the flat tables of a ragged launch: (int64 frame offsets, int32 geometry rows).

    frame_off : (B, n_t) element offsets of each clip's kept frames in the source buffer
    geom      : per clip (in_hw, resize_hw, window (top, left, out_h, out_w), hflip); every window is out_hw
    """
    offs = torch.as_tensor(frame_off, dtype=torch.int64)
    if offs.dim() != 2 or offs.shape[0] == 0 or offs.shape[1] == 0:
        raise RuntimeError("frame_off must be a non-empty (B, n_t) table")
    if len(geom) != offs.shape[0]:
        raise RuntimeError("geom needs one entry per clip (%d clips)" % offs.shape[0])
    rows = []
    for (ih, iw), (nh, nw), (top, left, oh, ow), flip in geom:
        if (oh, ow) != tuple(out_hw):
            raise RuntimeError("every crop window must be %s (got %s)" % (tuple(out_hw), (oh, ow)))
        rows += [int(ih), int(iw), int(nh), int(nw), int(top), int(left), 1 if flip else 0]
    return offs.contiguous().view(-1), torch.tensor(rows, dtype=torch.int32)


def clip_transform_ragged(src, frame_off, geom, out_hw, mean=None, std=None, div255=False, out_dtype=torch.float16,
                          slow_alpha=None):
    """The fused chain on a batch whose clips read frames of their own sizes, in one launch (pv_clip_transform_ragged).

    src       : flat uint8 or float32 CUDA tensor of packed (H, W, 3) frames, as ``decode_batch`` writes them
    frame_off : (B, n_t) element offsets of each clip's kept frames in src (an offset may repeat)
    geom      : per clip ((in_h, in_w), (new_h, new_w), (top, left, out_h, out_w), hflip)
    Returns (B, 3, n_t, out_h, out_w) of out_dtype, or [slow, fast] with ``slow_alpha``.
    """
    if not torch.is_tensor(src) or src.device.type != "cuda":
        raise RuntimeError("pytorchvideo_b200 transforms run on the GPU only (no CPU path)")
    if src.dtype not in (torch.uint8, torch.float32) or not src.is_contiguous():
        raise RuntimeError("the ragged source must be a contiguous uint8 or float32 tensor")
    if out_dtype not in (torch.float16, torch.float32):
        raise RuntimeError("the ragged mode writes float16 or float32")
    offs, rows = ragged_tables(frame_off, geom, out_hw)
    check_ragged_offsets(src, offs, geom)
    return launch_clip_ragged(src, offs.to(src.device), rows.to(src.device), rows, len(geom), out_hw, mean, std,
                              div255, out_dtype, slow_alpha)


def check_ragged_offsets(src, offs, geom):
    """Raise unless every frame of the flat offset table ``offs`` lies inside ``src``."""
    n_t = offs.numel() // len(geom)
    sizes = torch.tensor([g[0][0] * g[0][1] * 3 for g in geom], dtype=torch.int64).repeat_interleave(n_t)
    if int(offs.min()) < 0 or int((offs + sizes).max()) > src.numel():
        raise RuntimeError("a frame offset lies outside the source buffer")


def launch_clip_ragged(src, offs_d, rows_d, rows, B, out_hw, mean=None, std=None, div255=False,
                       out_dtype=torch.float16, slow_alpha=None):
    """The pv_clip_transform_ragged launch of ``clip_transform_ragged`` on tables already on the device and checked:
    ``offs_d`` / ``rows_d`` the device copies of ``ragged_tables``' offsets and rows, ``rows`` the host rows."""
    lib = L.load()
    dev = src.device
    n_t = offs_d.numel() // B
    oh, ow = (int(v) for v in out_hw)
    d = L.ClipBatchDesc()
    d.C, d.n_clips, d.n_t, d.out_h, d.out_w = 3, B, n_t, oh, ow
    _set_arith(d, 3, mean, std, div255)
    d.src_dtype, d.dst_dtype = _DT[src.dtype], _DT[out_dtype]
    out = torch.empty((B, 3, n_t, oh, ow), dtype=out_dtype, device=dev)
    d.d_clip = out.stride(0)
    slow_d, out_slow = None, None
    if slow_alpha is not None:
        slow_d, d.n_slow = _slow_table(n_t, slow_alpha, dev)
        out_slow = torch.empty((B, 3, d.n_slow, oh, ow), dtype=out_dtype, device=dev)
        d.d_slow_clip = out_slow.stride(0)
    L.check(lib.pv_clip_transform_ragged(C.byref(d), src.data_ptr(), offs_d.data_ptr(), rows_d.data_ptr(),
                                         rows.data_ptr(), slow_d.data_ptr() if slow_d is not None else None,
                                         out.data_ptr(), out_slow.data_ptr() if out_slow is not None else None,
                                         torch.cuda.current_stream(dev).cuda_stream), "pv_clip_transform_ragged")
    out._pv_keepalive = (offs_d, rows_d, slow_d)     # device tables must outlive the asynchronous launch
    return [out_slow, out] if slow_alpha is not None else out


# ---- reference-named functional API -----------------------------------------------------------
def _as_clip_batch(x, temporal_dim):
    """View an N-D tensor with its temporal dim at -3 as (clips, channels <= 4, T, H, W) without copying."""
    nd = x.dim()
    if nd < 3:
        raise RuntimeError("uniform_temporal_subsample needs at least (T, H, W)")
    td = temporal_dim % nd
    if td != nd - 3:
        raise NotImplementedError("only temporal_dim == -3 (…, T, H, W) has a B200 kernel; got dim %d of %d" % (temporal_dim, nd))
    lead = x.shape[:td]
    v = x.reshape((-1,) + tuple(x.shape[td:])) if nd != 4 else x      # (L, T, H, W); a view for contiguous leading dims
    Ld = v.shape[0]
    if Ld <= 4:
        return v.unsqueeze(0), lead                  # one clip of L channels
    return v.unsqueeze(1), lead                      # L clips of one channel


def uniform_temporal_subsample(x, num_samples, temporal_dim=-3):
    """functional.py:19-41 on any (…, T, H, W) tensor (4-D clips, 5-D batches as used with temporal_dim=2 by
    tests/test_models_slowfast.py:142-144): frame selection only, dtype preserved (uint8 stays uint8)."""
    if not torch.is_tensor(x) or x.device.type != "cuda":
        raise RuntimeError("pytorchvideo_b200 transforms run on the GPU only (no CPU path)")
    if x.dtype not in _DT:
        raise RuntimeError("unsupported clip dtype %s" % x.dtype)
    v, lead = _as_clip_batch(x, temporal_dim)
    idx = temporal_indices(v.shape[2], num_samples)
    out = clip_transform_batch(v, frame_idx=idx, out_dtype=x.dtype)
    return out.reshape(tuple(lead) + (int(idx.numel()),) + tuple(x.shape[-2:]))


def uniform_temporal_subsample_repeated(frames, frame_ratios, temporal_dim=-3):
    """functional.py:134-160: one subsampled tensor per ratio (SlowFast: frame_ratios=(alpha, 1))."""
    t = frames.shape[temporal_dim]
    return [uniform_temporal_subsample(frames, t // r, temporal_dim) for r in frame_ratios]


def short_side_scale(x, size, interpolation="bilinear", backend="pytorch"):
    assert len(x.shape) == 4
    assert x.dtype == torch.float32
    assert backend in ("pytorch", "opencv")
    if interpolation != "bilinear" or backend != "pytorch":
        raise NotImplementedError("only bilinear / pytorch semantics have a B200 kernel")
    return clip_transform(x, resize_hw=short_side_size(x.shape[2], x.shape[3], size))


def div_255(x):
    return clip_transform(x, div255=True)


def uniform_crop(images, size, spatial_idx):
    y, xo, h, w = uniform_crop_window(images.shape[2], images.shape[3], size, spatial_idx)
    return images[:, :, y:y + h, xo:xo + w]   # a view, exactly like the reference's slicing


# ---- RandomResizedCrop (functional.py random_resized_crop) --------------------------------------------------------
def random_resized_crop_window(scale, ratio, height, width, log_uniform_ratio=True, num_tries=10):
    """(top, left, h, w) of an Inception-style crop, drawn from torch's global RNG like the reference's
    _get_param_spatial_crop: up to num_tries (area, aspect ratio) draws, then a central crop."""
    assert num_tries >= 1, "num_tries must be at least 1"
    if scale[0] > scale[1]:
        scale = (scale[1], scale[0])
    if ratio[0] > ratio[1]:
        ratio = (ratio[1], ratio[0])
    for _ in range(num_tries):
        target_area = height * width * (scale[0] + torch.rand(1).item() * (scale[1] - scale[0]))
        if log_uniform_ratio:
            lo, hi = math.log(ratio[0]), math.log(ratio[1])
            aspect = math.exp(lo + torch.rand(1).item() * (hi - lo))
        else:
            aspect = ratio[0] + torch.rand(1).item() * (ratio[1] - ratio[0])
        w = int(round(math.sqrt(target_area * aspect)))
        h = int(round(math.sqrt(target_area / aspect)))
        if 0 < w <= width and 0 < h <= height:
            i = torch.randint(0, height - h + 1, (1,)).item()
            j = torch.randint(0, width - w + 1, (1,)).item()
            return i, j, h, w
    in_ratio = float(width) / float(height)
    if in_ratio < min(ratio):
        w, h = width, int(round(width / min(ratio)))
    elif in_ratio > max(ratio):
        h, w = height, int(round(height * max(ratio)))
    else:
        w, h = width, height
    return (height - h) // 2, (width - w) // 2, h, w


def random_resized_crop_boxes(t, height, width, scale, aspect_ratio, shift=False, log_uniform_ratio=True, num_tries=10):
    """Per-frame (top, left, h, w) of one clip of t frames: one window for every frame, or with ``shift`` a second
    window for the last frame and torch.linspace(...) + int() in between, as the reference."""
    assert scale[0] > 0 and scale[1] > 0, "min and max of scale range must be greater than 0"
    assert aspect_ratio[0] > 0 and aspect_ratio[1] > 0, "min and max of aspect_ratio range must be greater than 0"
    box = random_resized_crop_window(scale, aspect_ratio, height, width, log_uniform_ratio, num_tries)
    if not shift:
        return [box] * t
    box2 = random_resized_crop_window(scale, aspect_ratio, height, width, log_uniform_ratio, num_tries)
    cols = [[int(v) for v in torch.linspace(a, b, steps=t).tolist()] for a, b in zip(box, box2)]
    return list(zip(*cols))


def clip_transform_rrc(x, boxes, target_hw, frame_idx=None, flips=None, mean=None, std=None, div255=False,
                       out_dtype=torch.float32):
    """The batched chain in RandomResizedCrop mode (pv_clip_transform_rrc): frame selection, /255, normalisation and
    a per-(clip, kept frame) window resized to target_hw, then an optional per-clip horizontal flip, in ONE launch.

    x     : (B, 3, T, H, W) or (3, T, H, W) uint8 / float32 CUDA clip(s), any strides
    boxes : per clip, a list of (top, left, h, w) per kept frame
    flips : per clip bool (None = no flip)"""
    squeeze = torch.is_tensor(x) and x.dim() == 4
    if squeeze:
        x, boxes, flips = x.unsqueeze(0), [boxes], None if flips is None else [flips]
    if not torch.is_tensor(x) or x.dim() != 5:
        raise RuntimeError("expected a (B, C, T, H, W) or (C, T, H, W) tensor")
    if x.device.type != "cuda":
        raise RuntimeError("pytorchvideo_b200 transforms run on the GPU only (no CPU path)")
    if x.dtype not in (torch.uint8, torch.float32):
        raise RuntimeError("RandomResizedCrop reads uint8 or float32 clips (got %s)" % x.dtype)
    if out_dtype not in (torch.float16, torch.float32):
        raise RuntimeError("RandomResizedCrop writes float16 or float32 (got %s)" % out_dtype)
    B, Cc, T, H, W = x.shape
    if Cc != 3:
        raise RuntimeError("RandomResizedCrop needs 3-channel clips (got %d)" % Cc)
    idx = torch.arange(T) if frame_idx is None else torch.as_tensor(frame_idx).long().cpu()
    if idx.numel() == 0 or int(idx.min()) < 0 or int(idx.max()) >= T:
        raise RuntimeError("frame index out of range")
    n_t = int(idx.numel())
    oh, ow = int(target_hw[0]), int(target_hw[1])
    if len(boxes) != B or any(len(b) != n_t for b in boxes):
        raise RuntimeError("boxes needs one window per kept frame of every clip")
    flat = []
    for b in range(B):
        f = 1 if flips is not None and flips[b] else 0
        for top, left, h, w in boxes[b]:
            if top < 0 or left < 0 or h < 1 or w < 1 or top + h > H or left + w > W:
                raise RuntimeError("crop window (%d, %d, %d, %d) outside the %dx%d frame" % (top, left, h, w, H, W))
            flat += [int(top), int(left), int(h), int(w), f]
    lib = L.load()
    dev = x.device
    d = L.ClipBatchDesc()
    d.C, d.n_clips, d.n_t = Cc, B, n_t
    d.in_h, d.in_w, d.new_h, d.new_w = H, W, oh, ow
    d.out_h, d.out_w = oh, ow
    d.s_clip, d.sc, d.st, d.sh, d.sw = x.stride(0), x.stride(1), x.stride(2), x.stride(3), x.stride(4)
    normalize = mean is not None or std is not None
    mean_l = [float(m) for m in (mean if mean is not None else [0.0] * Cc)]
    std_l = [float(v) for v in (std if std is not None else [1.0] * Cc)]
    mean_l = mean_l * Cc if len(mean_l) == 1 else mean_l
    std_l = std_l * Cc if len(std_l) == 1 else std_l
    for i in range(4):
        d.mean[i] = mean_l[i] if i < len(mean_l) else 0.0
        d.stdv[i] = std_l[i] if i < len(std_l) else 1.0
    d.div255, d.normalize = 1 if div255 else 0, 1 if normalize else 0
    d.src_dtype, d.dst_dtype = _DT[x.dtype], _DT[out_dtype]
    out = torch.empty((B, Cc, n_t, oh, ow), dtype=out_dtype, device=dev)
    d.d_clip = out.stride(0)
    idx_d = _dev_i32(idx.tolist(), dev)
    boxes_d = torch.tensor(flat, dtype=torch.int32).to(dev)
    L.check(lib.pv_clip_transform_rrc(C.byref(d), x.data_ptr(), idx_d.data_ptr(), boxes_d.data_ptr(), out.data_ptr(),
                                      torch.cuda.current_stream(dev).cuda_stream), "pv_clip_transform_rrc")
    out._pv_keepalive = (idx_d, boxes_d)
    return out[0] if squeeze else out


def random_resized_crop(frames, target_height, target_width, scale, aspect_ratio, shift=False, log_uniform_ratio=True,
                        interpolation="bilinear", num_tries=10):
    """Reference functional.random_resized_crop on a float32 (C, T, H, W) CUDA clip, or a (B, C, T, H, W) batch with
    one independent draw per clip in clip order.  Bilinear only."""
    if interpolation != "bilinear":
        raise NotImplementedError("only bilinear RandomResizedCrop has a kernel (got %r)" % (interpolation,))
    if not torch.is_tensor(frames) or frames.dim() not in (4, 5):
        raise RuntimeError("expected a (C, T, H, W) or (B, C, T, H, W) tensor")
    if frames.device.type != "cuda":
        raise RuntimeError("pytorchvideo_b200 transforms run on the GPU only (no CPU path)")
    if frames.dtype != torch.float32:
        raise RuntimeError("random_resized_crop takes float32 clips (got %s)" % frames.dtype)
    x = frames.unsqueeze(0) if frames.dim() == 4 else frames
    T, H, W = x.shape[2], x.shape[3], x.shape[4]
    boxes = [random_resized_crop_boxes(T, H, W, scale, aspect_ratio, shift, log_uniform_ratio, num_tries)
             for _ in range(x.shape[0])]
    out = clip_transform_rrc(x, boxes, (target_height, target_width))
    return out[0] if frames.dim() == 4 else out


# ---- detection boxes (functional.py:195-445): pv_clip_boxes_transform ---------------------------------------------
# The box functions take (K, 4) (x1, y1, x2, y2) boxes as CUDA tensors, CPU tensors or numpy arrays (the reference's
# detection tutorial passes numpy).  Host boxes are copied to the clip's device, or to the current CUDA device when
# there is no clip, and every result is a CUDA tensor of the boxes' dtype (float32 or float64): the engine has no CPU
# path.  That is the one difference from the reference.
_BOX_DT = {torch.float32: L.BOX_F32, torch.float64: L.BOX_F64}


def _check_clip(images):
    if not torch.is_tensor(images) or images.dim() != 4:
        raise RuntimeError("expected a (C, T, H, W) clip")
    if images.device.type != "cuda":
        raise RuntimeError("pytorchvideo_b200 transforms run on the GPU only (no CPU path)")


def _boxes_on(boxes, dev=None):
    """``boxes`` as a contiguous (K, 4) float32 / float64 CUDA tensor on ``dev`` (default: its own CUDA device, or the
    current one for host boxes).  Returns the tensor itself when it already is one."""
    if isinstance(boxes, np.ndarray):
        boxes = torch.from_numpy(boxes)
    if not torch.is_tensor(boxes):
        raise RuntimeError("boxes must be a tensor or a numpy array (got %s)" % type(boxes).__name__)
    if boxes.dim() != 2 or boxes.shape[1] != 4:
        raise RuntimeError("boxes must be (K, 4) (x1, y1, x2, y2) rows (got shape %s)" % (tuple(boxes.shape),))
    if boxes.dtype not in _BOX_DT:
        raise RuntimeError("boxes must be float32 or float64 (got %s)" % boxes.dtype)
    if dev is None:
        dev = boxes.device if boxes.device.type == "cuda" else torch.device("cuda", torch.cuda.current_device())
    return boxes.to(dev).contiguous()


def _int_arg(v, what):
    if int(v) != v:
        raise RuntimeError("%s must be an integer (got %r)" % (what, v))
    return int(v)


def clip_boxes_transform(boxes, steps, in_hw=(0, 0), new_hw=(0, 0), offset=(0, 0), hflip=False, out_hw=(0, 0),
                         n_clips=1, box_start=None, geom=None, out=None, rois=False):
    """Run pv_clip_boxes_transform on a contiguous (K, 4) float32 / float64 CUDA tensor ``boxes``.

    steps   : mask of _lib.BOX_* steps, applied in the order CLIP_SRC, SCALE, CROP, CLIP_CROP, FLIP, CLIP_OUT
    in_hw   : source frame (CLIP_SRC; the scale factor is new / in of the short side's axis)
    new_hw, offset=(top, left), hflip : every clip's geometry, unless ``geom`` (device int32 [n_clips][6], the layout
              pv_clip_transform_batch reads) gives it per clip
    out_hw  : crop / output frame (CLIP_CROP, FLIP, CLIP_OUT)
    box_start: device int32 [n_clips + 1] offsets of each clip's boxes (None: one clip owns them all)
    out     : destination (K, 4) tensor of the boxes' dtype (None: a new tensor; ``boxes`` itself scales in place)
    Returns (out, rois): rois is the fp32 (K, 5) (clip, x1, y1, x2, y2) tensor when ``rois`` is set, else None."""
    dev = boxes.device
    K = int(boxes.shape[0])
    if out is None:
        out = torch.empty_like(boxes)
    r = torch.empty((K, 5), dtype=torch.float32, device=dev) if rois else None
    if K == 0:
        return out, r
    if box_start is None:
        if n_clips != 1:
            raise RuntimeError("box_start is needed for more than one clip")
        box_start = _dev_i32([0, K], dev)
    d = L.BoxesDesc()
    d.n_clips, d.n_boxes, d.steps, d.dtype = int(n_clips), K, int(steps), _BOX_DT[boxes.dtype]
    d.in_h, d.in_w = int(in_hw[0]), int(in_hw[1])
    d.new_h, d.new_w = int(new_hw[0]), int(new_hw[1])
    d.top, d.left, d.hflip = int(offset[0]), int(offset[1]), 1 if hflip else 0
    d.out_h, d.out_w = int(out_hw[0]), int(out_hw[1])
    L.check(L.load().pv_clip_boxes_transform(C.byref(d), boxes.data_ptr(), box_start.data_ptr(),
                                             geom.data_ptr() if geom is not None else None, out.data_ptr(),
                                             r.data_ptr() if r is not None else None,
                                             torch.cuda.current_stream(dev).cuda_stream), "pv_clip_boxes_transform")
    out._pv_keepalive = (boxes, box_start, geom)     # inputs must outlive the asynchronous launch
    return out, r


def clip_boxes_transform_ragged(boxes, steps, box_start, geom, geom_host, out_hw, out=None, rois=False):
    """Run pv_clip_boxes_transform_ragged: the boxes of clips with frames of their own sizes, in one launch.

    boxes    : contiguous (K, 4) float32 / float64 CUDA tensor
    steps    : mask of _lib.BOX_* steps; BOX_DENORM (x * in_w, y * in_h) runs first, then the others in their order
    box_start: device int32 [n_clips + 1] offsets of each clip's boxes
    geom     : device int32 [n_clips][7] {in_h, in_w, new_h, new_w, top, left, hflip}, the table
               ``clip_transform_ragged`` reads (``ragged_tables``' rows); ``geom_host`` the same table on the host
    out_hw   : crop / output frame of every clip
    Returns (out, rois) as ``clip_boxes_transform`` does."""
    dev = boxes.device
    K = int(boxes.shape[0])
    geom_host = geom_host.to(torch.int32).contiguous()
    n_clips = geom_host.numel() // 7
    if geom_host.device.type != "cpu" or geom_host.numel() != 7 * n_clips or n_clips < 1:
        raise RuntimeError("geom_host must be a host table of 7 ints per clip")
    if out is None:
        out = torch.empty_like(boxes)
    r = torch.empty((K, 5), dtype=torch.float32, device=dev) if rois else None
    d = L.BoxesDesc()
    d.n_clips, d.n_boxes, d.steps, d.dtype = n_clips, K, int(steps), _BOX_DT[boxes.dtype]
    d.out_h, d.out_w = int(out_hw[0]), int(out_hw[1])
    L.check(L.load().pv_clip_boxes_transform_ragged(C.byref(d), boxes.data_ptr(), box_start.data_ptr(),
                                                    geom.data_ptr(), geom_host.data_ptr(), out.data_ptr(),
                                                    r.data_ptr() if r is not None else None,
                                                    torch.cuda.current_stream(dev).cuda_stream),
            "pv_clip_boxes_transform_ragged")
    out._pv_keepalive = (boxes, box_start, geom)     # inputs must outlive the asynchronous launch
    return out, r


def short_side_scale_with_boxes(images, boxes, size, interpolation="bilinear", backend="pytorch"):
    """functional.py:195-230: the clip's short side scaled to ``size`` (short_side_scale) and the boxes multiplied by
    the same factor, in place when ``boxes`` is a CUDA tensor (the reference's ``boxes *=``).  Returns (images, boxes)."""
    _check_clip(images)
    _, _, h, w = images.shape
    b = _boxes_on(boxes, images.device)
    images = short_side_scale(images, size, interpolation, backend)
    _, _, new_h, new_w = images.shape
    res, _ = clip_boxes_transform(b, L.BOX_SCALE, in_hw=(h, w), new_hw=(new_h, new_w), out=b)
    if torch.is_tensor(boxes) and boxes.device == b.device and b is not boxes:
        boxes.copy_(b)               # a non-contiguous CUDA view: write the result back into it
        res = boxes
    return images, res


def random_short_side_scale_with_boxes(images, boxes, min_size, max_size, interpolation="bilinear",
                                       backend="pytorch"):
    """functional.py:233-264: the short side drawn with torch.randint(min_size, max_size + 1) (torch's global RNG)."""
    size = torch.randint(min_size, max_size + 1, (1,)).item()
    return short_side_scale_with_boxes(images, boxes, size, interpolation, backend)


def random_crop_offsets(height, width, size):
    """The offsets random_crop_with_boxes draws (functional.py:284-293): numpy's global RNG, exclusive upper bound,
    y first and each only when that side is longer than ``size``.  None when the frame already is size x size (the
    reference then returns the clip alone and draws nothing)."""
    if height == size and width == size:
        return None
    y = int(np.random.randint(0, height - size)) if height > size else 0
    x = int(np.random.randint(0, width - size)) if width > size else 0
    return y, x


def _crop_boxes_of(cropped, b, y, x):
    out, _ = clip_boxes_transform(b, L.BOX_CROP | L.BOX_CLIP_CROP, offset=(y, x), out_hw=tuple(cropped.shape[-2:]))
    return out


def random_crop_with_boxes(images, size, boxes):
    """functional.py:267-299.  Returns (cropped view, boxes) - or ``images`` alone, as the reference does, when the
    clip already is size x size."""
    _check_clip(images)
    b = _boxes_on(boxes, images.device)      # argument checks before any draw
    yx = random_crop_offsets(images.shape[2], images.shape[3], size)
    if yx is None:
        return images
    y, x = yx
    cropped = images[:, :, y:y + size, x:x + size]
    return cropped, _crop_boxes_of(cropped, b, y, x)


def uniform_crop_with_boxes(images, size, spatial_idx, boxes):
    """functional.py:350-377: the uniform_crop window (a view) and the boxes cropped, then clipped to it."""
    _check_clip(images)
    y, x, _, _ = uniform_crop_window(images.shape[2], images.shape[3], size, spatial_idx)
    if y < 0 or x < 0:
        raise RuntimeError("crop size %d larger than the %dx%d frame" % (size, images.shape[2], images.shape[3]))
    cropped = images[:, :, y:y + size, x:x + size]
    return cropped, _crop_boxes_of(cropped, _boxes_on(boxes, images.device), y, x)


def horizontal_flip_with_boxes(prob, images, boxes):
    """functional.py:380-404: flips when np.random.uniform() < prob (numpy's global RNG, drawn on every call).  The
    clip is mirrored by the batched transform kernel with identity geometry (dtype preserved); the boxes become
    x1' = (W - x2) - 1, x2' = (W - x1) - 1.  Returns (images, a new boxes tensor)."""
    _check_clip(images)
    b = _boxes_on(boxes, images.device)
    flip = np.random.uniform() < prob
    if flip:
        images = clip_transform_batch(images, hflip=True, out_dtype=images.dtype)
    out, _ = clip_boxes_transform(b, L.BOX_FLIP if flip else 0, hflip=flip, out_hw=tuple(images.shape[-2:]))
    return images, out


def clip_boxes_to_image(boxes, height, width):
    """functional.py:407-426: x to [0, width - 1], y to [0, height - 1] (numpy's minimum / maximum)."""
    b = _boxes_on(boxes)
    out, _ = clip_boxes_transform(b, L.BOX_CLIP_OUT, out_hw=(_int_arg(height, "height"), _int_arg(width, "width")))
    return out


def crop_boxes(boxes, x_offset, y_offset):
    """functional.py:429-445: x - x_offset, y - y_offset."""
    b = _boxes_on(boxes)
    out, _ = clip_boxes_transform(b, L.BOX_CROP, offset=(_int_arg(y_offset, "y_offset"), _int_arg(x_offset, "x_offset")))
    return out
