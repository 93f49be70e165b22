"""Golden vectors of the baseline-JPEG decoder and FrameVideo (tests/golden/jpeg.pt).

Encodes seeded content (smooth gradients and uniform noise) with Pillow and OpenCV into fixtures covering 4:2:0,
4:2:2, 4:4:0, 4:4:4 and grayscale, sizes from 1x1 to 257x341, qualities 50-100, optimised Huffman tables, restart
intervals, and APPn / COM / EXIF segments; plus fixtures the decoder must reject (progressive, CMYK, EXIF
orientation 6).  For each decodable fixture it stores ``cv2.cvtColor(cv2.imdecode(b, IMREAD_COLOR), BGR2RGB)`` and
asserts that Pillow gives the same bytes, and torchvision's CPU decode_jpeg too except on 4:4:0 (its libjpeg
upsamples 1x2 chroma by replication, without libjpeg-turbo's fancy h1v2 filter).

It then writes a 12-frame directory (names frame_1.jpg .. frame_12.jpg, so that natural order differs from the
lexicographic one) and runs the reference's FrameVideo.from_directory(...).get_clip at several (start, end,
frame_filter), storing values, dtype, shape, strides and frame_indices (None for the out-of-range starts,
"ValueError" where the range holds no frame).

    PYTHONPATH=<reference checkout> python oracle/gen_golden_jpeg.py
"""
import io
import os
import sys
import tempfile
import types

import cv2
import numpy as np
import torch
import torchvision
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))

GOLD = os.path.join(ROOT, "tests", "golden", "jpeg.pt")

# frame_filter names the tests can rebuild
FILTERS = {None: None, "every2": lambda ix: ix[::2], "first3": lambda ix: ix[:3]}
CLIP_CASES = [(0.0, 0.5, None), (0.15, 1.0, None), (0.25, 10.0, "every2"), (0.0, 1.2, "first3"), (1.2, 2.0, None),
              (0.05, 0.95, "every2"), (-0.1, 0.5, None), (1.3, 2.0, None)]
CLIP_FPS = 10.0


def content(h, w, kind, seed):
    r = np.random.default_rng(seed)
    if kind == "noise":
        return r.integers(0, 256, (h, w, 3), dtype=np.uint8)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.stack([x * 255 / max(w - 1, 1), y * 255 / max(h - 1, 1),
                    (x + y) * 127 / max(w + h - 2, 1) + 60 * np.sin(x / 5.0) + 60], -1)
    return np.clip(img + r.normal(0, 6, img.shape), 0, 255).astype(np.uint8)


def pil(img, **kw):
    bio = io.BytesIO()
    Image.fromarray(img).save(bio, "JPEG", **kw)
    return bio.getvalue()


def cv(img, *params):
    ok, buf = cv2.imencode(".jpg", img[..., ::-1] if img.ndim == 3 else img, list(params))
    assert ok
    return buf.tobytes()


def exif(orientation):
    ex = Image.Exif()
    ex[0x0112] = orientation
    return ex.tobytes()


def fixtures():
    """[(name, bytes, expected)]: expected "ok" or the name of the rejection class"""
    out = []
    add = lambda name, b, exp="ok": out.append((name, b, exp))
    add("s420_smooth_q95_opt_257x341", pil(content(257, 341, "smooth", 1), quality=95, subsampling=2, optimize=True))
    add("s422_noise_q50_257x341", pil(content(257, 341, "noise", 2), quality=50, subsampling=1))
    add("s444_smooth_q100_33x47", pil(content(33, 47, "smooth", 3), quality=100, subsampling=0))
    add("s444_noise_q100_40x56", pil(content(40, 56, "noise", 4), quality=100, subsampling=0))
    add("s420_noise_q100_24x40", pil(content(24, 40, "noise", 5), quality=100, subsampling=2))
    add("s422_smooth_q75_opt_64x48", pil(content(64, 48, "smooth", 6), quality=75, subsampling=1, optimize=True))
    add("s440_smooth_q85_48x64", cv(content(48, 64, "smooth", 7), cv2.IMWRITE_JPEG_QUALITY, 85,
                                    cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440))
    add("s440_noise_q95_17x9", cv(content(17, 9, "noise", 8), cv2.IMWRITE_JPEG_QUALITY, 95,
                                  cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440))
    add("gray_smooth_q75_9x17", cv(content(9, 17, "smooth", 9)[..., 0], cv2.IMWRITE_JPEG_QUALITY, 75))
    add("gray_noise_q95_61x83", pil(content(61, 83, "noise", 10)[..., 0], quality=95))
    add("gray_1x1", pil(content(1, 1, "noise", 11)[..., 0], quality=90))
    add("s420_1x1", pil(content(1, 1, "noise", 12), quality=90, subsampling=2))
    add("s444_1x1", pil(content(1, 1, "noise", 13), quality=90, subsampling=0))
    add("s420_smooth_q90_9x17", pil(content(9, 17, "smooth", 14), quality=90, subsampling=2))
    add("s422_noise_q90_17x9", pil(content(17, 9, "noise", 15), quality=90, subsampling=1))
    add("s420_noise_q90_2x3", pil(content(2, 3, "noise", 16), quality=90, subsampling=2))      # chroma 2 wide
    add("s422_noise_q90_3x4", pil(content(3, 4, "noise", 17), quality=90, subsampling=1))
    add("s420_smooth_q90_rst2_120x160", cv(content(120, 160, "smooth", 18), cv2.IMWRITE_JPEG_QUALITY, 90,
                                           cv2.IMWRITE_JPEG_RST_INTERVAL, 2))
    add("s444_noise_q90_rst1_37x53", cv(content(37, 53, "noise", 19), cv2.IMWRITE_JPEG_QUALITY, 90,
                                        cv2.IMWRITE_JPEG_RST_INTERVAL, 1,
                                        cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444))
    add("gray_noise_q80_rst3_33x65", cv(content(33, 65, "noise", 20)[..., 0], cv2.IMWRITE_JPEG_QUALITY, 80,
                                       cv2.IMWRITE_JPEG_RST_INTERVAL, 3))
    add("s420_smooth_q90_app_com_exif1_40x40", pil(content(40, 40, "smooth", 21), quality=90, subsampling=2,
                                                   comment=b"frame 7 of a test clip", exif=exif(1),
                                                   icc_profile=b"\0" * 300))
    add("progressive", pil(content(32, 32, "smooth", 22), quality=90, progressive=True), "progressive")
    bio = io.BytesIO()
    Image.fromarray(content(16, 16, "smooth", 23)).convert("CMYK").save(bio, "JPEG", quality=90)
    add("cmyk", bio.getvalue(), "colorspace")
    add("exif_orientation6", pil(content(16, 24, "smooth", 24), quality=90, exif=exif(6)), "orientation")
    return out


def cv2_rgb(b):
    return cv2.cvtColor(cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2RGB)


def load_reference_frame_video():
    """The reference's data/frame_video.py without running data/__init__.py (which imports every dataset and
    PyAV): a bare `pytorchvideo.data` package over the reference directory, and a PyAV stand-in exposing the one
    name data/utils.py reads at import."""
    import pytorchvideo
    pkg = types.ModuleType("pytorchvideo.data")
    pkg.__path__ = [os.path.join(os.path.dirname(pytorchvideo.__file__), "data")]
    sys.modules["pytorchvideo.data"] = pkg
    av = types.ModuleType("av")
    av.video = types.ModuleType("av.video")
    av.video.frame = types.ModuleType("av.video.frame")
    av.video.frame.PictureType = type("PictureType", (), {})
    sys.modules.update({"av": av, "av.video": av.video, "av.video.frame": av.video.frame})
    from pytorchvideo.data.frame_video import FrameVideo
    return FrameVideo


def main():
    fx = fixtures()
    names, blobs, expected, decoded = [], [], [], []
    for name, b, exp in fx:
        names.append(name)
        blobs.append(torch.frombuffer(bytearray(b), dtype=torch.uint8))
        expected.append(exp)
        if exp != "ok":
            decoded.append(None)
            continue
        ref = cv2_rgb(b)
        p = np.asarray(Image.open(io.BytesIO(b)).convert("RGB"))
        t = torchvision.io.decode_jpeg(torch.frombuffer(bytearray(b), dtype=torch.uint8),
                                       mode=torchvision.io.ImageReadMode.RGB).permute(1, 2, 0).numpy()
        assert np.array_equal(ref, p), name
        assert np.array_equal(ref, t) or name.startswith("s440"), name
        decoded.append(torch.from_numpy(ref.copy()))

    FrameVideo = load_reference_frame_video()
    frame_names = ["frame_%d.jpg" % (i + 1) for i in range(12)]
    frame_blobs = [pil(content(24, 32, "smooth", 100 + i), quality=90, subsampling=2) for i in range(12)]
    clips = []
    with tempfile.TemporaryDirectory() as td:
        vdir = os.path.join(td, "video_a")
        os.makedirs(vdir)
        for n, b in zip(frame_names, frame_blobs):
            open(os.path.join(vdir, n), "wb").write(b)
        video = FrameVideo.from_directory(vdir, fps=CLIP_FPS)
        assert video.name == "video_a"
        for start, end, filt in CLIP_CASES:
            try:
                r = video.get_clip(start, end, FILTERS[filt])
            except ValueError:          # no frame in range: np.stack([]) in the reference's loader
                clips.append("ValueError")
                continue
            if r is None:
                clips.append(None)
                continue
            v = r["video"]
            clips.append({"video": v.contiguous(), "dtype": str(v.dtype), "shape": tuple(v.shape),
                          "stride": tuple(v.stride()), "frame_indices": list(r["frame_indices"]),
                          "audio": r["audio"]})
        duration = video.duration
    torch.save({"names": names, "blobs": blobs, "expected": expected, "decoded": decoded,
                "frame_names": frame_names, "frame_blobs": [torch.frombuffer(bytearray(b), dtype=torch.uint8)
                                                            for b in frame_blobs],
                "clip_fps": CLIP_FPS, "clip_cases": CLIP_CASES, "clips": clips, "duration": duration,
                "versions": {"cv2": cv2.__version__, "PIL": Image.__version__, "torchvision": torchvision.__version__}},
               GOLD)
    print("wrote", GOLD, os.path.getsize(GOLD), "bytes,", sum(e == "ok" for e in expected), "decodable fixtures")


if __name__ == "__main__":
    main()
