"""CPU: the baseline-JPEG host parser (pv_jpeg_parse) and FrameVideo's index rules, against tests/golden/jpeg.pt."""
import ctypes
import os
import struct
import subprocess
import tempfile

import pytest
import torch

from pytorchvideo_b200 import _lib as L
from pytorchvideo_b200.data import FrameVideo, decode_jpeg_frames, parse_jpeg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "jpeg.pt"), weights_only=False)
ZIGZAG = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
          21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53,
          60, 61, 54, 47, 55, 62, 63]
OK = [(n, bytes(b.numpy().tobytes()), d) for n, b, e, d in zip(GOLD["names"], GOLD["blobs"], GOLD["expected"],
                                                                 GOLD["decoded"]) if e == "ok"]
MODES = {"gray": L.JPEG_GRAY, "s444": L.JPEG_H1V1, "s422": L.JPEG_H2V1, "s440": L.JPEG_H1V2, "s420": L.JPEG_H2V2}


def markers(b):
    """[(marker, payload)] up to and including SOS, walked independently of the library"""
    out, p = [], 2
    while p < len(b):
        assert b[p] == 0xFF
        while b[p] == 0xFF:
            p += 1
        m = b[p]
        n = struct.unpack(">H", b[p + 1:p + 3])[0]
        out.append((m, b[p + 3:p + 1 + n]))
        p += 1 + n
        if m == 0xDA:
            return out, p
    raise AssertionError("no SOS")


def canonical(bits, vals):
    """{(length, code): symbol} of a DHT table"""
    codes, code = {}, 0
    k = 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            codes[(length, code)] = vals[k]
            code += 1
            k += 1
        code <<= 1
    return codes


@pytest.mark.parametrize("name,blob,dec", OK, ids=[o[0] for o in OK])
def test_parse_geometry_tables_and_segments(name, blob, dec):
    rc, f, batch, segs = parse_jpeg(blob)
    assert rc == 0, L.last_error()
    H, W = dec.shape[:2]
    assert (f.height, f.width) == (H, W)
    assert f.mode == MODES[name.split("_")[0]]
    ms, scan_start = markers(blob)
    sof = [p for m, p in ms if m in (0xC0, 0xC1)][0]
    nc = sof[5]
    assert f.ncomp == nc
    hv = [(sof[7 + 3 * c] >> 4, sof[7 + 3 * c] & 15) for c in range(nc)]
    if nc == 3:
        hmax, vmax = max(h for h, _ in hv), max(v for _, v in hv)
        assert [(f.h[c], f.v[c]) for c in range(3)] == hv
        assert (f.mcus_x, f.mcus_y) == (-(-W // (8 * hmax)), -(-H // (8 * vmax)))
        assert [f.bw[c] for c in range(3)] == [f.mcus_x * h for h, _ in hv]
        assert [f.dw[c] for c in range(3)] == [-(-W * h // hmax) for h, _ in hv]
        assert [f.dh[c] for c in range(3)] == [-(-H * v // vmax) for _, v in hv]
    else:
        assert (f.mcus_x, f.mcus_y) == (-(-W // 8), -(-H // 8))
    assert f.n_blocks == sum(f.bw[c] * f.bh[c] for c in range(nc))
    assert batch.ws_bytes == 192 * f.n_blocks and batch.out_elems == 3 * H * W
    # quantisation tables, natural order
    qts = {}
    for m, p in ms:
        if m == 0xDB:
            i = 0
            while i < len(p):
                pq, tq = p[i] >> 4, p[i] & 15
                vals = [p[i + 1 + k] for k in range(64)] if pq == 0 else \
                    [struct.unpack(">H", p[i + 1 + 2 * k:i + 3 + 2 * k])[0] for k in range(64)]
                nat = [0] * 64
                for k in range(64):
                    nat[ZIGZAG[k]] = vals[k]
                qts[tq] = nat
                i += 1 + 64 * (pq + 1)
    for c in range(nc):
        assert list(f.qt[c]) == qts[sof[8 + 3 * c]]
    # Huffman lookup tables: every code of <= 9 bits fills its prefix range with (length, symbol)
    for m, p in ms:
        if m == 0xC4:
            i = 0
            while i < len(p):
                tc, th = p[i] >> 4, p[i] & 15
                bits = list(p[i + 1:i + 17])
                vals = list(p[i + 17:i + 17 + sum(bits)])
                t = (f.dc if tc == 0 else f.ac)[th]
                for (length, code), sym in canonical(bits, vals).items():
                    if length <= 9:
                        for k in range(1 << (9 - length)):
                            assert t.look[(code << (9 - length)) + k] == (length << 8) | sym
                    else:
                        assert t.maxcode[length] >= code and t.val[code + t.valoff[length]] == sym
                i += 17 + sum(bits)
    # restart interval and segment ranges
    dri = [p for m, p in ms if m == 0xDD]
    ri = struct.unpack(">H", dri[0])[0] if dri else 0
    assert f.restart_interval == ri
    assert "rst" in name or ri == 0
    total = f.mcus_x * f.mcus_y
    assert f.n_segments == len(segs) == (-(-total // ri) if ri else 1)
    assert segs[0][0] == scan_start
    for k, (b0, b1) in enumerate(segs):
        assert b0 <= b1 <= len(blob)
        if k > 0:
            assert blob[b0 - 2] == 0xFF and blob[b0 - 1] == 0xD0 + ((k - 1) & 7)
    assert blob[segs[-1][1]:segs[-1][1] + 2] == b"\xff\xd9"


def _sof(marker, prec=8, h=16, w=16, comps=((1, 0x22, 0), (2, 0x11, 0), (3, 0x11, 0))):
    body = bytes([prec]) + struct.pack(">HHB", h, w, len(comps)) + b"".join(bytes(c) for c in comps)
    return b"\xff\xd8" + b"\xff" + bytes([marker]) + struct.pack(">H", 2 + len(body)) + body


@pytest.mark.parametrize("blob,code", [
    (_sof(0xC9), "arithmetic"),
    (_sof(0xCA), "arithmetic"),
    (_sof(0xC2), "progressive"),
    (_sof(0xC3), "lossless"),
    (_sof(0xC5), "hierarchical"),
    (_sof(0xC0, prec=12), "precision"),
    (_sof(0xC1, prec=12), "precision"),
    (_sof(0xC0, h=0), "dnl"),
    (_sof(0xC0, comps=((1, 0x11, 0), (2, 0x11, 0))), "components"),
    (_sof(0xC0, comps=((1, 0x11, 0),) * 5), "components"),
    (_sof(0xC0, comps=((1, 0x11, 0),) * 4), "colorspace"),
    (_sof(0xC0, comps=((1, 0x41, 0), (2, 0x11, 0), (3, 0x11, 0))), "sampling"),
], ids=["sof9", "sof10", "sof2", "sof3", "sof5", "p12", "p12_sof1", "dnl_height", "two_comps", "five_comps", "four_comps",
        "h4v1"])
def test_rejected_classes_have_their_own_codes(blob, code):
    # the sampling check runs once the scan header is known: give those headers the tables and SOS they need
    if code == "sampling":
        dqt = b"\xff\xdb\x00\x43\x00" + bytes([1] * 64)
        dht = b"\xff\xc4" + struct.pack(">H", 2 + 17 + 1) + b"\x00" + bytes([1] + [0] * 15) + b"\x00"
        dht += b"\xff\xc4" + struct.pack(">H", 2 + 17 + 1) + b"\x10" + bytes([1] + [0] * 15) + b"\x00"
        sos = b"\xff\xda\x00\x0c\x03\x01\x00\x02\x00\x03\x00\x00\x3f\x00"
        blob = blob + dqt + dht + sos + b"\x00\xff\xd9"
    rc = parse_jpeg(blob)[0]
    assert L.JPEG_ERRORS.get(rc) == code, (rc, L.last_error())


def test_rejected_fixtures():
    for n, b, e in zip(GOLD["names"], GOLD["blobs"], GOLD["expected"]):
        if e != "ok":
            assert L.JPEG_ERRORS.get(parse_jpeg(b)[0]) == e, n


def _with_dnl_or_second_scan(blob, tail):
    """blob with `tail` inserted between the entropy data and EOI"""
    assert blob.endswith(b"\xff\xd9")
    return blob[:-2] + tail + b"\xff\xd9"


def test_multiscan_and_dnl_markers_after_the_scan():
    blob = OK[0][1]
    assert L.JPEG_ERRORS.get(parse_jpeg(_with_dnl_or_second_scan(blob, b"\xff\xdc\x00\x04\x01\x01"))[0]) == "dnl"
    sos = markers(blob)[0][-1][1]
    second = b"\xff\xda" + struct.pack(">H", 2 + len(sos)) + sos + b"\x00"
    assert L.JPEG_ERRORS.get(parse_jpeg(_with_dnl_or_second_scan(blob, second))[0]) == "multiscan"
    # a scan of one of three components is a multi-scan (non-interleaved) file
    ms, start = markers(blob)
    p = blob.index(b"\xff\xda")
    one = b"\xff\xda\x00\x08\x01\x01\x00\x00\x3f\x00"
    assert L.JPEG_ERRORS.get(parse_jpeg(blob[:p] + one + blob[start:])[0]) == "multiscan"


def test_truncated_headers_and_scans_are_invalid():
    for name, blob, _ in OK[:6] + [o for o in OK if "rst" in o[0]][:1] + [o for o in OK if "app" in o[0]]:
        _, scan_start = markers(blob)
        for cut in list(range(0, scan_start, 7)) + [scan_start, scan_start + 1]:
            assert parse_jpeg(blob[:cut])[0] == -1, (name, cut)
        # entropy data without a closing marker runs off the buffer
        assert parse_jpeg(blob[:-2])[0] == -1, name
    assert parse_jpeg(b"")[0] == -1 and parse_jpeg(b"\xff\xd8")[0] == -1 and parse_jpeg(b"GIF89a")[0] == -1


def test_batch_appends_frames():
    lib = L.load()
    blobs = [OK[0][1], OK[8][1], OK[-2][1]]
    cap = sum(len(b) for b in blobs)
    segs = (ctypes.c_uint32 * (2 * cap))()
    batch = L.JpegBatch()
    frames = (L.JpegFrame * 3)()
    seen = []
    for i, b in enumerate(blobs):
        before = (batch.data_bytes, batch.n_segments, batch.n_blocks, batch.out_elems)
        assert lib.pv_jpeg_parse(b, len(b), ctypes.byref(batch), ctypes.byref(frames[i]), segs, cap) == 0
        f = frames[i]
        assert (f.data_off, f.seg_base, f.block_base, f.out_off) == before
        seen.append(f.mode)
    assert batch.n_frames == 3 and batch.mode_mask == sum(1 << m for m in set(seen))
    assert batch.max_blocks == max(f.n_blocks for f in frames)
    assert batch.max_pixels == max(f.width * f.height for f in frames)
    # a rejected stream leaves the batch as it was
    state = bytes(batch)
    bad = (L.JpegFrame)()
    assert lib.pv_jpeg_parse(b"\xff\xd8", 2, ctypes.byref(batch), ctypes.byref(bad), segs, cap) == -1
    assert bytes(batch) == state


def test_struct_sizes_match_header():
    probe = r'''
    #include <stdio.h>
    #include "pv_b200.h"
    int main(){ printf("%zu %zu %zu\n", sizeof(pv_jpeg_huff), sizeof(pv_jpeg_frame), sizeof(pv_jpeg_batch)); return 0; }'''
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "p.c")
        open(c, "w").write(probe)
        exe = os.path.join(td, "p")
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe], check=True)
        sizes = [int(v) for v in subprocess.run([exe], capture_output=True, text=True).stdout.split()]
    assert sizes == [ctypes.sizeof(L.JpegHuff), ctypes.sizeof(L.JpegFrame), ctypes.sizeof(L.JpegBatch)]


def _frame_dir(td):
    vdir = os.path.join(td, "video_a")
    os.makedirs(vdir)
    for n, b in zip(GOLD["frame_names"], GOLD["frame_blobs"]):
        open(os.path.join(vdir, n), "wb").write(b.numpy().tobytes())
    return vdir


FILTERS = {None: None, "every2": lambda ix: ix[::2], "first3": lambda ix: ix[:3]}


def test_frame_video_index_rules_match_the_reference():
    with tempfile.TemporaryDirectory() as td:
        vdir = _frame_dir(td)
        cache = {}
        v = FrameVideo.from_directory(vdir, fps=GOLD["clip_fps"], path_order_cache=cache)
        # natural order: frame_2 before frame_10, unlike a plain sort
        assert [os.path.basename(p) for p in cache[vdir]] == ["frame_%d.jpg" % (i + 1) for i in range(12)]
        assert sorted(os.listdir(vdir)) != [os.path.basename(p) for p in cache[vdir]]
        assert v.name == "video_a" and v.duration == GOLD["duration"]
        # the cache answers without listing the directory again
        cache[vdir] = cache[vdir][:4]
        assert FrameVideo.from_directory(vdir, fps=GOLD["clip_fps"], path_order_cache=cache).duration == 4 / GOLD["clip_fps"]
        for (start, end, filt), want in zip(GOLD["clip_cases"], GOLD["clips"]):
            got = v.frame_indices(start, end, FILTERS[filt])
            if want is None:
                assert got is None
            elif want == "ValueError":
                assert got == []
                with pytest.raises(ValueError):
                    v.get_clip(start, end, FILTERS[filt])
            else:
                assert got == want["frame_indices"]
                assert want["audio"] is None
    with pytest.raises(AssertionError):
        FrameVideo.from_frame_paths([])
    with pytest.raises(AssertionError):
        FrameVideo(1.0, 30.0)
    assert FrameVideo(2.0, 30.0, video_frame_to_path_fn=lambda i: "/x/clip_b/%d.jpg" % i).name == "clip_b"


def test_product_has_no_cpu_path():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError):
        decode_jpeg_frames([OK[0][1]])
    with tempfile.TemporaryDirectory() as td:
        v = FrameVideo.from_directory(_frame_dir(td), fps=GOLD["clip_fps"])
        with pytest.raises(RuntimeError):
            v.get_clip(0.0, 0.5)


def test_size_and_table_slot_limits_are_unsupported():
    gray = lambda h, w: _sof(0xC0, h=h, w=w, comps=((1, 0x11, 0),))
    assert parse_jpeg(gray(65535, 65535))[0] == -3          # 4.3e9 pixels: the batch's pixel counts are int
    assert parse_jpeg(gray(46341, 46341))[0] == -3          # just above 2^31 - 1
    assert parse_jpeg(gray(46340, 46340))[0] == -1          # fits; then the stream is truncated
    dht2 = b"\xff\xc4" + struct.pack(">H", 2 + 17 + 1) + b"\x02" + bytes([1] + [0] * 15) + b"\x00"
    assert parse_jpeg(b"\xff\xd8" + dht2)[0] == -3          # Huffman table slot 2 (SOF1 allows 0..3)


HOST_HARNESS = r'''
#include "pv_jpeg.cu"
#include <vector>
namespace pv {
void set_error(const char*, ...) {}
void count_launch(const char*) {}
}
using namespace pv::jpeg;
// Decodes one stream with the kernels' __host__ __device__ routines, in the kernels' order, on the CPU.
int main(int argc, char** argv) {
  FILE* fp = fopen(argv[1], "rb");
  std::vector<uint8_t> d(1 << 22);
  const long long n = (long long)fread(d.data(), 1, d.size(), fp);
  fclose(fp);
  pv_jpeg_batch b = {};
  pv_jpeg_frame* f = new pv_jpeg_frame();
  std::vector<uint32_t> segs(2 * (n / 2 + 2));
  if (pv_jpeg_parse(d.data(), n, &b, f, segs.data(), n / 2 + 2)) return 2;
  std::vector<int16_t> coef(b.n_blocks * 64);
  std::vector<uint8_t> planes(b.n_blocks * 64), out(3ll * f->width * f->height);
  alignas(16) int16_t blk[64];
  for (int s = 0; s < f->n_segments; ++s)
    if (decode_segment(*f, f->dc, f->ac, segs.data(), d.data(), s, coef.data(), blk, kNaturalOrderHost)) return 3;
  for (int i = 0; i < f->n_blocks; ++i) {
    const int c = f->ncomp == 3 && i >= f->block_off[2] ? 2 : f->ncomp == 3 && i >= f->block_off[1] ? 1 : 0;
    const int local = i - f->block_off[c], by = local / f->bw[c], bx = local % f->bw[c];
    int ws[64];
    for (int k = 0; k < 8; ++k) idct_col(coef.data() + i * 64, f->qt[c], k, ws);
    for (int k = 0; k < 8; ++k)
      idct_row(ws, k, planes.data() + f->block_off[c] * 64 + (by * 8 + k) * f->bw[c] * 8 + bx * 8);
  }
  for (int y = 0; y < f->height; ++y)
    for (int x = 0; x < f->width; ++x) {
      uint8_t* o = out.data() + 3ll * (y * f->width + x);
      switch (f->mode) {
        case PV_JPEG_GRAY: pixel_rgb<PV_JPEG_GRAY>(*f, planes.data(), x, y, o); break;
        case PV_JPEG_H1V1: pixel_rgb<PV_JPEG_H1V1>(*f, planes.data(), x, y, o); break;
        case PV_JPEG_H2V1: pixel_rgb<PV_JPEG_H2V1>(*f, planes.data(), x, y, o); break;
        case PV_JPEG_H1V2: pixel_rgb<PV_JPEG_H1V2>(*f, planes.data(), x, y, o); break;
        default: pixel_rgb<PV_JPEG_H2V2>(*f, planes.data(), x, y, o); break;
      }
    }
  fp = fopen(argv[2], "wb");
  fwrite(out.data(), 1, out.size(), fp);
  fclose(fp);
  return 0;
}
'''


def test_decoder_routines_match_cv2_on_the_cpu():
    """The entropy, IDCT and colour routines the kernels call are __host__ __device__: compiled for the host, they
    must give cv2's bytes on every golden fixture (no GPU needed)."""
    from pytorchvideo_b200 import _build
    nvcc = _build._nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    with tempfile.TemporaryDirectory() as td:
        src = os.path.join(td, "harness.cu")
        open(src, "w").write(HOST_HARNESS)
        exe = os.path.join(td, "harness")
        subprocess.run([nvcc, "-std=c++17", "-O2", "-gencode", _build.ARCH, "-diag-suppress", "550",
                        "-I", os.path.join(ROOT, "pytorchvideo_b200", "csrc"), "-o", exe, src], check=True)
        for name, blob, dec in OK:
            jpg, rgb = os.path.join(td, "in.jpg"), os.path.join(td, "out.rgb")
            open(jpg, "wb").write(blob)
            assert subprocess.run([exe, jpg, rgb]).returncode == 0, name
            got = torch.frombuffer(bytearray(open(rgb, "rb").read()), dtype=torch.uint8).view(dec.shape)
            assert torch.equal(got, dec), name
