"""GPU: the batched baseline-JPEG decoder and FrameVideo, bit for bit against cv2 / the reference (tests/golden/jpeg.pt)."""
import os
import tempfile

import pytest
import torch

from pytorchvideo_b200 import _lib as L
from pytorchvideo_b200.data import FrameVideo, decode_jpeg_frames, parse_jpeg
from pytorchvideo_b200.data.jpeg import decode_batch
from pytorchvideo_b200.transforms import functional as Fv

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "jpeg.pt"), weights_only=False)
OK = [(n, bytes(b.numpy().tobytes()), d) for n, b, e, d in zip(GOLD["names"], GOLD["blobs"], GOLD["expected"],
                                                                 GOLD["decoded"]) if e == "ok"]
MODE_NAME = {L.JPEG_GRAY: "gray", L.JPEG_H1V1: "h1v1", L.JPEG_H2V1: "h2v1", L.JPEG_H1V2: "h1v2", L.JPEG_H2V2: "h2v2"}
FILTERS = {None: None, "every2": lambda ix: ix[::2], "first3": lambda ix: ix[:3]}


def _delta(before):
    after = L.kernel_counts()
    return {k: v - before.get(k, 0) for k, v in after.items() if v != before.get(k, 0)}


@pytest.mark.parametrize("name,blob,dec", OK, ids=[o[0] for o in OK])
def test_fixture_bit_exact_u8_and_f32(name, blob, dec):
    mode = parse_jpeg(blob)[1].mode
    before = L.kernel_counts()
    got = decode_jpeg_frames([blob])
    torch.cuda.synchronize()
    assert _delta(before) == {"jpeg_huffman_kernel": 1, "jpeg_idct_islow_kernel": 1,
                              "jpeg_ycc_rgb_kernel<%s,u8>" % MODE_NAME[mode]: 1}
    assert got.shape == (1,) + tuple(dec.shape) and got.dtype == torch.uint8 and got.is_cuda
    assert torch.equal(got[0].cpu(), dec)
    before = L.kernel_counts()
    got32 = decode_jpeg_frames([torch.frombuffer(bytearray(blob), dtype=torch.uint8)], out_dtype=torch.float32)
    assert _delta(before)["jpeg_ycc_rgb_kernel<%s,f32>" % MODE_NAME[mode]] == 1
    assert got32.dtype == torch.float32 and torch.equal(got32[0].cpu(), dec.float())


def test_one_launch_mixes_modes_restarts_and_sizes():
    blobs = [b for _, b, _ in OK]
    modes = {parse_jpeg(b)[1].mode for b in blobs}
    assert len(modes) == 5 and any("rst" in n for n, _, _ in OK)
    before = L.kernel_counts()
    flat, sizes = decode_batch(blobs)
    torch.cuda.synchronize()
    want = {"jpeg_huffman_kernel": 1, "jpeg_idct_islow_kernel": 1}
    want.update({"jpeg_ycc_rgb_kernel<%s,u8>" % MODE_NAME[m]: 1 for m in modes})
    assert _delta(before) == want
    flat = flat.cpu()
    pos = 0
    for (name, blob, dec), (h, w) in zip(OK, sizes):
        assert (h, w) == tuple(dec.shape[:2])
        got = flat[pos:pos + h * w * 3].view(h, w, 3)
        assert torch.equal(got, dec), name
        assert torch.equal(got, decode_jpeg_frames([blob])[0].cpu()), name
        pos += h * w * 3
    assert pos == flat.numel()


def test_decode_into_a_clip_buffer_and_repeatability():
    blobs = [b.numpy().tobytes() for b in GOLD["frame_blobs"]]
    clip = torch.full((len(blobs), 24, 32, 3), 7, dtype=torch.uint8, device="cuda")
    assert decode_jpeg_frames(blobs, out=clip) is clip
    again = decode_jpeg_frames(blobs)
    assert torch.equal(clip, again)
    assert torch.equal(decode_jpeg_frames(blobs), again)
    with pytest.raises(RuntimeError):
        decode_jpeg_frames([OK[0][1], OK[2][1]])          # two sizes in one call
    # an out of the right element count but the wrong shape is refused before anything is written
    wrong = torch.full((len(blobs), 32, 24, 3), 7, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError, match="out is"):
        decode_jpeg_frames(blobs, out=wrong)
    torch.cuda.synchronize()
    assert bool((wrong == 7).all())


def _frame_dir(td):
    vdir = os.path.join(td, "video_a")
    os.makedirs(vdir)
    for n, b in zip(GOLD["frame_names"], GOLD["frame_blobs"]):
        open(os.path.join(vdir, n), "wb").write(b.numpy().tobytes())
    return vdir


@pytest.mark.parametrize("multithreaded_io", [False, True])
def test_frame_video_get_clip_matches_the_reference(multithreaded_io):
    with tempfile.TemporaryDirectory() as td:
        v = FrameVideo.from_directory(_frame_dir(td), fps=GOLD["clip_fps"], multithreaded_io=multithreaded_io)
        for (start, end, filt), want in zip(GOLD["clip_cases"], GOLD["clips"]):
            if want == "ValueError":
                with pytest.raises(ValueError):
                    v.get_clip(start, end, FILTERS[filt])
                continue
            got = v.get_clip(start, end, FILTERS[filt])
            if want is None:
                assert got is None
                continue
            video = got["video"]
            assert video.is_cuda and str(video.dtype) == want["dtype"]
            assert tuple(video.shape) == want["shape"] and tuple(video.stride()) == want["stride"]
            assert got["frame_indices"] == want["frame_indices"] and got["audio"] is None
            assert torch.equal(video.cpu(), want["video"])


def test_decode_then_clip_transform_equals_the_transform_of_the_reference_frames():
    want_clip = GOLD["clips"][1]                 # frames 2..9 decoded by the reference, (C, T, H, W) float32
    idx = want_clip["frame_indices"]
    blobs = [GOLD["frame_blobs"][i].numpy().tobytes() for i in idx]
    dec = decode_jpeg_frames(blobs)                                        # (T, H, W, 3) uint8
    ref = want_clip["video"].to(torch.uint8).permute(1, 2, 3, 0).contiguous().cuda()
    kw = dict(frame_idx=[0, 2, 4, 6], resize_hw=(36, 48), window=(6, 8, 24, 32), mean=(0.45, 0.45, 0.45),
              std=(0.225, 0.225, 0.225), div255=True, out_dtype=torch.float16)
    got = Fv.clip_transform_batch(dec.permute(3, 0, 1, 2), **kw)
    want = Fv.clip_transform_batch(ref.permute(3, 0, 1, 2), **kw)
    assert torch.equal(got, want)


def _scan_bounds(blob):
    seg = parse_jpeg(blob)[3]
    return seg[0][0], seg[-1][1]


def test_corrupt_entropy_data_names_the_frame_and_the_stream_recovers():
    name, blob, dec = OK[0]
    b0, b1 = _scan_bounds(blob)
    truncated = blob[:b0 + (b1 - b0) // 2] + b"\xff\xd9"
    # 64 one-bits in the middle of the scan: no JPEG Huffman code is all ones
    mid = (b0 + b1) // 2
    flipped = blob[:mid] + b"\xff\x00" * 8 + blob[mid + 16:]
    assert parse_jpeg(truncated)[0] == 0 and parse_jpeg(flipped)[0] == 0
    with pytest.raises(RuntimeError, match=r"frame 1: corrupt JPEG entropy data \(.*overrun"):
        decode_jpeg_frames([blob, truncated, blob])
    with pytest.raises(RuntimeError, match=r"frame 2: corrupt JPEG entropy data \(bad Huffman code"):
        decode_jpeg_frames([blob, blob, flipped])
    # a restart marker out of sequence
    rn, rblob, rdec = [o for o in OK if "rst" in o[0] and o[0].startswith("s420")][0]
    segs = parse_jpeg(rblob)[3]
    p = segs[2][0] - 1
    bad_rst = rblob[:p] + bytes([0xD0 + ((rblob[p] - 0xD0 + 3) & 7)]) + rblob[p + 1:]
    with pytest.raises(RuntimeError, match=r"frame 0: corrupt JPEG entropy data \(.*restart marker"):
        decode_jpeg_frames([bad_rst, rblob])
    # a header the parser rejects names its frame too
    with pytest.raises(RuntimeError, match=r"frame 1: JPEG rejected \(invalid\)"):
        decode_jpeg_frames([blob, blob[:100]])
    # later decodes on the same stream are unaffected
    assert torch.equal(decode_jpeg_frames([blob, blob])[1].cpu(), dec)
    assert torch.equal(decode_jpeg_frames([rblob])[0].cpu(), rdec)
