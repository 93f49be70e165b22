"""Batched baseline-JPEG decode on the GPU (pv_jpeg_parse / pv_jpeg_decode), bit for bit what
``cv2.cvtColor(cv2.imdecode(buf, cv2.IMREAD_COLOR), cv2.COLOR_BGR2RGB)`` returns (data/frame_video.py:242-245)."""
import ctypes as C
import threading

import numpy as np
import torch

from .. import _lib as L

# pinned staging buffer per device, reused across calls: a call holds the lock until it has read the status back,
# which waits for the host-to-device copy
_STAGE = {}
_STAGE_LOCK = threading.Lock()


def _as_bytes(frame):
    if isinstance(frame, (bytes, bytearray, memoryview)):
        return np.frombuffer(frame, dtype=np.uint8)
    if torch.is_tensor(frame):
        if frame.dtype != torch.uint8 or frame.dim() != 1:
            raise RuntimeError("a frame tensor must be 1-D uint8")
        return frame.detach().cpu().contiguous().numpy()
    raise RuntimeError("a frame must be bytes or a 1-D uint8 tensor, got %s" % type(frame).__name__)


def _parse_error(name, rc):
    kind = L.JPEG_ERRORS.get(rc, "invalid" if rc == -1 else "unsupported" if rc == -3 else "status %d" % rc)
    return RuntimeError("%s: JPEG rejected (%s): %s" % (name, kind, L.last_error()))


def parse_jpeg(data):
    """Host parse of one stream: (rc, pv_jpeg_frame, pv_jpeg_batch, [(begin, end) byte range of each segment]).
    rc is 0 or the code pv_jpeg_parse returned (a pv_jpeg_error per rejected class, -1 for malformed data)."""
    buf = np.ascontiguousarray(_as_bytes(data))
    cap = buf.size // 2 + 2
    segs = np.zeros(2 * cap, dtype=np.uint32)
    batch, frame = L.JpegBatch(), L.JpegFrame()
    rc = L.load().pv_jpeg_parse(buf.ctypes.data, buf.size, C.byref(batch), C.byref(frame), segs.ctypes.data, cap)
    n = batch.n_segments if rc == 0 else 0
    return rc, frame, batch, [(int(segs[2 * k]), int(segs[2 * k + 1])) for k in range(n)]


def decode_batch(frames, out=None, out_dtype=torch.uint8, same_size=False, out_shape=None, names=None):
    """Decode JPEG streams of any sizes with one host-to-device copy and one launch sequence.

    Returns (out, [(H, W) per frame]); out is flat and holds frame i's (H, W, 3) pixels right after frame i-1's.
    ``out`` may be given as a contiguous CUDA tensor of out_dtype with exactly that many elements.  same_size
    raises on the first frame whose size differs from frame 0's; with it, out_shape (the caller's view of out) must be
    (N, H, W, 3) of the parsed frames, checked before anything is written.  Errors name frame i as names[i] when
    ``names`` is given (e.g. the file paths), else as "frame i".
    """
    if out_dtype not in (torch.uint8, torch.float32):
        raise RuntimeError("out_dtype must be torch.uint8 or torch.float32")
    if len(frames) == 0:
        raise RuntimeError("no frames to decode")
    lib = L.load()
    L.require_device()
    dev = out.device if out is not None else torch.device("cuda", torch.cuda.current_device())
    bufs = [_as_bytes(f) for f in frames]
    n = len(bufs)
    data_bytes = sum(b.size for b in bufs)
    # staging layout: [streams back to back | frames | segment pairs]; pv_jpeg_parse places stream i at data_off =
    # the bytes of the streams before it, and the parse reads it from there
    frames_off = (data_bytes + 15) // 16 * 16
    segs_off = frames_off + n * C.sizeof(L.JpegFrame)
    cap = data_bytes // 2 + 2 * n
    with _STAGE_LOCK:
        host = _STAGE.get(dev.index)
        if host is None or host.numel() < segs_off + 8 * cap:
            host = _STAGE[dev.index] = torch.empty(max(segs_off + 8 * cap, 1 << 20), dtype=torch.uint8,
                                                   pin_memory=True)
        base = host.data_ptr()
        pos = 0
        for b in bufs:
            C.memmove(base + pos, b.ctypes.data, b.size)
            pos += b.size
        batch = L.JpegBatch()
        farr = (L.JpegFrame * n).from_address(base + frames_off)
        sizes = []
        for i, b in enumerate(bufs):
            rc = lib.pv_jpeg_parse(base + batch.data_bytes, b.size, C.byref(batch), C.byref(farr[i]),
                                   base + segs_off, cap)
            if rc != 0:
                raise _parse_error(names[i] if names is not None else "frame %d" % i, rc)
            sizes.append((farr[i].height, farr[i].width))
            if same_size and sizes[i] != sizes[0]:
                raise RuntimeError("frame %d is %dx%d, frame 0 is %dx%d: all frames must share one size"
                                   % (i, sizes[i][1], sizes[i][0], sizes[0][1], sizes[0][0]))
        if same_size and out_shape is not None and tuple(out_shape) != (n,) + sizes[0] + (3,):
            raise RuntimeError("out is %s, the frames are (%d, %d, %d, 3)" % ((tuple(out_shape), n) + sizes[0]))
        if out is None:
            out = torch.empty(batch.out_elems, dtype=out_dtype, device=dev)
        elif (not out.is_cuda or out.dtype != out_dtype or not out.is_contiguous()
              or out.numel() != batch.out_elems):
            raise RuntimeError("out must be a contiguous %s CUDA tensor of %d elements (the frames are %s)"
                               % (out_dtype, batch.out_elems, sizes if not same_size else (n,) + sizes[0] + (3,)))
        staged = segs_off + 8 * batch.n_segments
        ws_off = (staged + 255) // 256 * 256
        st_off = ws_off + (batch.ws_bytes + 15) // 16 * 16
        dbuf = torch.empty(st_off + 4 * n, dtype=torch.uint8, device=dev)
        dbuf[:staged].copy_(host[:staged], non_blocking=True)
        d = dbuf.data_ptr()
        L.check(lib.pv_jpeg_decode(C.byref(batch), d + frames_off, d + segs_off, d, d + ws_off, batch.ws_bytes,
                                   out.data_ptr(), L.PV_U8 if out_dtype == torch.uint8 else L.PV_F32, d + st_off,
                                   torch.cuda.current_stream(dev).cuda_stream), "pv_jpeg_decode")
        status = dbuf[st_off:].view(torch.int32).cpu()
    bad = status.nonzero().flatten().tolist()
    if bad:
        s = int(status[bad[0]])
        why = [w for bit, w in ((L.JPEG_BAD_CODE, "bad Huffman code"), (L.JPEG_BAD_OVERRUN, "entropy data overrun"),
                                (L.JPEG_BAD_RESTART, "restart marker out of sequence")) if s & bit]
        name = names[bad[0]] if names is not None else "frame %d" % bad[0]
        raise RuntimeError("%s: corrupt JPEG entropy data (%s)" % (name, ", ".join(why)))
    return out, sizes


def decode_jpeg_frames(frames, out=None, out_dtype=torch.uint8):
    """Decode a batch of same-size JPEG frames to a (N, H, W, 3) CUDA tensor (uint8, or float32 holding 0..255).

    frames : sequence of ``bytes`` or 1-D uint8 tensors (whole JPEG files)
    out    : optional contiguous (N, H, W, 3) CUDA tensor of out_dtype to decode into, e.g. a clip buffer
    The streams are staged in one pinned buffer, copied with one host-to-device copy and decoded by one launch
    sequence on the current stream; the call returns once the per-frame status has been read back.  A frame the
    decoder rejects or finds corrupt raises RuntimeError naming its index, and so do frames of different sizes.
    """
    frames = list(frames)
    if out is not None and (out.dim() != 4 or out.shape[0] != len(frames) or out.shape[3] != 3):
        raise RuntimeError("out must be (N, H, W, 3) with N = %d" % len(frames))
    flat, sizes = decode_batch(frames, out=None if out is None else out.view(-1), out_dtype=out_dtype, same_size=True,
                               out_shape=None if out is None else out.shape)
    return out if out is not None else flat.view(len(frames), sizes[0][0], sizes[0][1], 3)
