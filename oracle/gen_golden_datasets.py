"""Golden vectors of the frame-folder datasets and clip samplers (tests/golden/datasets.pt).

Encodes seeded content with OpenCV into four frame folders of different (odd) sizes, some with restart markers, and
writes the index files the datasets read: a Charades frame csv, the SSv2 label json, video json and frame csv, a
Kinetics-style ``<path> <label>`` csv (with one encoded-video path and one unlabelled line), and a class-directory
tree of video files.  The fixture bytes are stored; the tests write them out again.

It then runs the reference's datasets on them under fixed ``torch`` and ``random`` seeds and stores every sample:
all keys, the ``"video"`` clip (uint8, its values are whole numbers) and the frame indices ``FrameVideo.get_clip``
loaded for it.  Each run is at ``num_workers=0``; two runs again in a DataLoader with two workers and a
SequentialSampler.  Last, the reference's clip samplers over a grid of durations and arguments.

    PYTHONPATH=<reference checkout> python oracle/gen_golden_datasets.py
"""
import json
import os
import random
import sys
import tempfile
from fractions import Fraction

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))

GOLD = os.path.join(ROOT, "tests", "golden", "datasets.pt")

# (name, frames, height, width, quality, restart interval in MCU rows (0: none))
VIDEOS = [("vid0", 12, 23, 31, 90, 0), ("vid1", 9, 30, 40, 90, 1), ("vid2", 15, 17, 45, 85, 0),
          ("vid3", 10, 26, 26, 95, 2)]

# sampler grid: (class name in clip_sampling, constructor arguments); durations each is run over
SAMPLERS = [("UniformClipSampler", (0.5,)), ("UniformClipSampler", (Fraction(2, 3), 0.25)),
            ("UniformClipSampler", (1.0, 0.4, True)), ("UniformClipSampler", (0.3, None, True, 1e-6)),
            ("UniformClipSampler", (Fraction(4, 30), Fraction(2, 30), False)),
            ("UniformClipSamplerTruncateFromStart", (0.5, None, False, 1e-6, 1.1)),
            ("RandomClipSampler", (0.5,)), ("RandomMultiClipSampler", (0.4, 3)),
            ("RandomMultiClipSamplerTruncateFromStart", (0.4, 2, 0.8)),
            ("ConstantClipsPerVideoSampler", (0.5, 3)), ("ConstantClipsPerVideoSampler", (0.4, 2, 3)),
            ("ConstantClipsPerVideoSampler", (2.0, 4))]
DURATIONS = [Fraction(1, 3), 0.5, 1.0, 1.3, 2.05, 10.0]
MAKE = [("uniform", (0.75,)), ("random", (0.75,)), ("constant_clips_per_video", (0.75, 2)), ("random_multi", (0.75, 2))]


def frame(h, w, t, seed):
    r = np.random.default_rng(seed * 1000 + t)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.stack([(x + 3 * t) * 255 / max(w - 1, 1), y * 255 / max(h - 1, 1),
                    60 * np.sin((x + y + 2 * t) / 4.0) + 120], -1)
    return np.clip(img + r.normal(0, 8, img.shape), 0, 255).astype(np.uint8)


def encode(img, quality, rst):
    params = [cv2.IMWRITE_JPEG_QUALITY, quality]
    if rst:
        params += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst * ((img.shape[1] + 15) // 16)]
    ok, buf = cv2.imencode(".jpg", img[..., ::-1], params)
    assert ok
    return buf.tobytes()


def fixture_files():
    """{relative path: bytes} of the whole fixture tree."""
    files = {}
    rng = random.Random(7)
    charades = ["original_vido_id video_id frame_id path labels"]
    for vi, (name, n, h, w, q, rst) in enumerate(VIDEOS):
        for t in range(n):
            rel = "frames/%s/frame_%d.jpg" % (name, t + 1)     # natural order differs from the lexicographic one
            files[rel] = encode(frame(h, w, t, vi), q, rst)
            labels = ",".join(str(rng.randrange(157)) for _ in range(rng.randrange(3)))
            charades.append('%s %d %d %s "%s"' % (name, vi, t, rel, labels))
    files["charades.csv"] = ("\n".join(charades) + "\n").encode()
    files["ssv2.csv"] = files["charades.csv"]
    files["ssv2_labels.json"] = json.dumps({"Pushing something": "0", "Dropping something into something": "1",
                                            "Holding something": "2"}).encode()
    files["ssv2_train.json"] = json.dumps([
        {"id": "vid2", "template": "Dropping [something] into [something]"},
        {"id": "missing", "template": "Holding [something]"},
        {"id": "vid0", "template": "Pushing [something]"},
        {"id": "vid3", "template": "Holding [something]"},
        {"id": "vid1", "template": "Pushing [something]"}]).encode()
    files["kinetics.csv"] = b"frames/vid0 3\nframes/vid1 0\nclips/bad.mp4 2\nframes/vid2 1\nframes/vid3\n"
    files["clips/bad.mp4"] = b"\x00\x00\x00\x18ftypmp42"
    for rel in ("classes/jump/a.mp4", "classes/jump/sub/b.avi", "classes/run/c.MP4", "classes/run/d.avi"):
        files[rel] = b"\x00\x00\x00\x18ftypmp42"
    files["classes/run/notes.txt"] = b"not a video\n"
    return files


def write_tree(root, files):
    for rel, data in files.items():
        path = os.path.join(root, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "wb") as f:
            f.write(data)


def datasets(root, D):
    """{run name: builder of the reference dataset from a video sampler class}."""
    csv = os.path.join(root, "charades.csv")
    ssv2 = [os.path.join(root, n) for n in ("ssv2_labels.json", "ssv2_train.json", "ssv2.csv")]
    kin = os.path.join(root, "kinetics.csv")
    return {
        "charades_uniform": lambda vs: D.Charades(csv, D.UniformClipSampler(Fraction(1, 5)), vs,
                                                  video_path_prefix=root, frames_per_clip=4),
        "charades_constant": lambda vs: D.Charades(csv, D.clip_sampling.ConstantClipsPerVideoSampler(0.1, 2, 2), vs,
                                                   video_path_prefix=root),
        "ssv2_random": lambda vs: D.SSv2(*ssv2, D.RandomClipSampler(0.2), vs, video_path_prefix=root,
                                         frames_per_clip=5, rand_sample_frames=True),
        "ssv2_middle": lambda vs: D.SSv2(*ssv2, D.UniformClipSampler(0.2), vs, video_path_prefix=root,
                                         frames_per_clip=3),
        "kinetics_random": lambda vs: D.Kinetics(kin, D.RandomClipSampler(0.25), vs, video_path_prefix=root,
                                                 decode_audio=False),
        "labeled_uniform_backpad": lambda vs: D.labeled_video_dataset(
            kin, D.UniformClipSampler(Fraction(4, 30), None, True), vs, video_path_prefix=root, decode_audio=False),
        "kinetics_decode_audio_default": lambda vs: D.Kinetics(kin, D.RandomClipSampler(0.25), vs,
                                                               video_path_prefix=root),
    }


# (run, video sampler): the worker-free runs; RandomSampler takes the torch seed (Charades, SSv2) or its own generator
RUNS0 = [("charades_uniform", "random"), ("charades_constant", "sequential"), ("ssv2_random", "random"),
         ("ssv2_middle", "sequential"), ("kinetics_random", "random"), ("labeled_uniform_backpad", "sequential"),
         ("kinetics_decode_audio_default", "sequential")]
RUNS2 = [("charades_uniform", "sequential"), ("kinetics_random", "sequential")]
SEED = 1234


def record(sample, indices):
    out = {k: v for k, v in sample.items() if k != "video"}
    v = sample["video"]
    assert torch.equal(v, v.round()) and v.min() >= 0 and v.max() <= 255
    out["video"] = v.to(torch.uint8).contiguous()
    out["frame_indices"] = indices
    return out


def run_dataset(ds, num_workers, log):
    torch.manual_seed(SEED)
    random.seed(SEED)
    if num_workers == 0:
        it = iter(ds)
        out = []
        while True:
            try:
                s = next(it)
            except StopIteration:
                return out
            except RuntimeError as e:
                return out + [{"error": str(e)}]
            out.append(record(s, list(log[-1])))
    loader = torch.utils.data.DataLoader(ds, batch_size=None, num_workers=num_workers)
    return [record(s, None) for s in loader]


def main():
    from pytorchvideo import data as D
    from pytorchvideo.data import clip_sampling as CS
    from pytorchvideo.data import frame_video as FV
    from pytorchvideo.data.labeled_video_paths import LabeledVideoPaths

    files = fixture_files()
    log = []
    get_clip = FV.FrameVideo.get_clip

    def logged_get_clip(self, *a, **k):
        res = get_clip(self, *a, **k)
        log.append(res["frame_indices"] if res is not None else None)
        return res

    FV.FrameVideo.get_clip = logged_get_clip
    samplers = {"random": torch.utils.data.RandomSampler, "sequential": torch.utils.data.SequentialSampler}
    gold = {"files": files, "seed": SEED, "runs0": {}, "runs2": {}}
    with tempfile.TemporaryDirectory() as root:
        write_tree(root, files)
        build = datasets(root, D)
        for name, vs in RUNS0:
            gold["runs0"][name] = {"sampler": vs, "samples": run_dataset(build[name](samplers[vs]), 0, log)}
        for name, vs in RUNS2:
            gold["runs2"][name] = {"sampler": vs, "samples": run_dataset(build[name](samplers[vs]), 2, log)}
        lp = LabeledVideoPaths.from_directory(os.path.join(root, "classes"))
        gold["class_directory"] = [(os.path.relpath(lp[i][0], root), lp[i][1]) for i in range(len(lp))]
        lp = LabeledVideoPaths.from_path(os.path.join(root, "kinetics.csv"))
        gold["csv_paths"] = [lp[i] for i in range(len(lp))]

    grid = []
    for k, (cls, args) in enumerate(SAMPLERS):
        for dur in DURATIONS:
            for first in (None, 0.0):
                random.seed(k)
                s = getattr(CS, cls)(*args)
                last, clips = first, []
                for _ in range(40):
                    c = s(last, dur, {})
                    clips.append(tuple(c))
                    last = c.clip_end_sec
                    done = c.is_last_clip[-1] if isinstance(c.is_last_clip, list) else c.is_last_clip
                    if done:
                        break
                grid.append(((cls, args), dur, first, clips))
    gold["samplers"] = grid
    gold["make_clip_sampler"] = [(kind, args, type(CS.make_clip_sampler(kind, *args)).__name__) for kind, args in MAKE]
    torch.save(gold, GOLD)
    n = sum(len(r["samples"]) for r in gold["runs0"].values()) + sum(len(r["samples"]) for r in gold["runs2"].values())
    print("wrote %s: %d dataset samples, %d sampler sequences, %d bytes" % (GOLD, n, len(grid), os.path.getsize(GOLD)))


if __name__ == "__main__":
    main()
