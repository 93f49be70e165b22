"""Golden vectors of the AVA dataset (tests/golden/ava.pt).

Encodes seeded content with OpenCV into three frame folders of different sizes (one portrait), and writes the files
the reference's ``Ava`` reads: a frame-paths file (one video listed out of frame_id order, one listed in part and
with a row from another directory), labels csvs of both row types, and a ``.pbtxt`` label map.  The rows cover
seconds outside [902, 1798] (as ints and as floats), an empty action label, boxes that collide under "%.2f", a
keyframe the label map prunes to nothing, boxes on the frame edges, and keyframes whose window starts before 0 s.
The fixture bytes are stored; the tests write them out again.

It then runs the reference's parsers and ``Ava`` (under the ``iopath`` / ``av`` shims) with a uniform and with a
random clip sampler, each with and without the label map, and stores every sample: all keys but the clip, and the
frame indices ``FrameVideo.get_clip`` loaded for it.  Each video's frames are stored once, as the reference decodes
them; every sample's clip is checked here to be those frames at its indices.  Last, ``TimeStampClipSampler`` windows
over a grid of durations (float and Fraction) and keyframe seconds.

    PYTHONPATH=<reference checkout> python oracle/gen_golden_ava.py
"""
import os
import sys
import tempfile
from fractions import Fraction

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.gen_golden_datasets import encode, frame, write_tree  # noqa: E402  (also puts the shims on sys.path)

GOLD = os.path.join(ROOT, "tests", "golden", "ava.pt")

# (name, frames, height, width, frame file name pattern); 100 frames at 30 fps reach keyframe second 903
VIDEOS = [("vidA", 100, 23, 31, "img_%05d.jpg"), ("vidB", 96, 33, 21, "img_%05d.jpg"),
          ("vidC", 100, 19, 27, "frame_%d.jpg")]

TRAIN_CSV = """vidA,0902,0.1,0.2,0.5,0.9,12,0
vidA,0901,0.1,0.2,0.5,0.9,12,0
vidA,0902,0.1,0.2,0.5,0.9,17,0
vidA,0902,0.104,0.2,0.5,0.9,80,1
vidA,0902,0.6,0.1,0.95,0.7,,2
vidA,1799,0.6,0.1,0.95,0.7,12,2
vidA,0903,0.3,0.3,0.6,0.6,99,3
vidB,0902,0.05,0.1,0.4,0.8,1,0
vidB,0902,0.5,0.2,1.0,1.0,5,1
vidB,901.9,0.5,0.2,1.0,1.0,5,1
vidB,902.0,0.05,0.1,0.4,0.8,2,0
vidB,0903,0.0,0.0,1.0,1.0,12,2
vidC,0903,0.2,0.25,0.7,0.75,2,0
vidC,1798.5,0.2,0.25,0.7,0.75,2,0
vidC,0902,0.9,0.9,1.0,1.0,17,1
vidC,0902,0.0,0.45,0.125,0.55,,4
"""

DET_CSV = """vidA,0902,0.1,0.2,0.5,0.9,,0.98
vidA,0903,0.2,0.1,0.7,0.8,12,0.91
vidA,0903,0.2049,0.1,0.7,0.8,80,0.55
vidA,0903,0.0,0.5,0.33,1.0,1,0.5
vidB,0902,0.3,0.3,0.9,0.95,1,0.77
vidB,0903,0.1,0.1,0.3,0.5,99,0.6
vidB,0903,0.5,0.5,0.9,0.9,,0.4
vidB,0900,0.5,0.5,0.9,0.9,2,0.4
vidC,0903,0.0,0.0,0.5,0.5,5,0.85
vidC,0903,0.5,0.5,1.0,1.0,17,0.125
"""

LABEL_MAP = """item {
  name: "bend/bow (at the waist)"
  id: 1
}
item {
  name: "crawl"
  label_id: 2
}
item {
  name: "dance"
  id: 5
}
item {
  name: "stand"
  id: 12
}
item {
  name: "walk"
  label_id: 17
}
item {
  name: "talk to (e.g., self, a person, a group)"
  id: 80
}
"""

# (run, clip sampler, video sampler, labels csv, with the label map)
RUNS = [("uniform", ("UniformClipSampler", (Fraction(1, 3),)), "sequential", "ava_train.csv", False),
        ("uniform_map", ("UniformClipSampler", (Fraction(1, 3),)), "sequential", "ava_train.csv", True),
        ("random", ("RandomClipSampler", (4.2,)), "random", "ava_det.csv", False),
        ("random_map", ("RandomClipSampler", (4.2,)), "random", "ava_det.csv", True)]
SEED = 4321
DURATIONS = [0.5, 4.2, Fraction(1, 3), Fraction(32, 30), 2]
KEYFRAMES = [2.0, 3.0, 897.0, 0.5]


def fixture_files():
    """{relative path: bytes} of the whole fixture tree."""
    files = {}
    rows = {}
    for vi, (name, n, h, w, pattern) in enumerate(VIDEOS):
        rows[name] = []
        for t in range(n):
            rel = "frames/%s/%s" % (name, pattern % (t + 1))
            files[rel] = encode(frame(h, w, t, 10 + vi), 90, 0)
            rows[name].append('%s %d %d %s ""' % (name, vi, t, rel))
    listed = rows["vidA"] + rows["vidB"][::-1] + rows["vidC"][:10]
    # a row of another directory with a later frame_id: the video's directory is its first frame's, by frame_id
    listed.append('vidC 2 500 frames/vidA/img_00001.jpg ""')
    files["ava_frame_list.csv"] = ("original_vido_id video_id frame_id path labels\n" + "\n".join(listed) + "\n").encode()
    files["ava_train.csv"] = TRAIN_CSV.encode()
    files["ava_det.csv"] = DET_CSV.encode()
    files["ava_label_map.pbtxt"] = LABEL_MAP.encode()
    return files


def plain(d):
    """Nested defaultdicts as dicts."""
    return {k: plain(v) for k, v in d.items()} if isinstance(d, dict) else d


def main():
    from pytorchvideo import data as D
    from pytorchvideo.data import ava as A
    from pytorchvideo.data import clip_sampling as CS
    from pytorchvideo.data import frame_video as FV

    files = fixture_files()
    log = []
    get_clip = FV.FrameVideo.get_clip

    def logged_get_clip(self, *a, **k):
        res = get_clip(self, *a, **k)
        log.append((a[:2], res["frame_indices"] if res is not None else None))
        return res

    FV.FrameVideo.get_clip = logged_get_clip
    samplers = {"random": torch.utils.data.RandomSampler, "sequential": torch.utils.data.SequentialSampler}
    gold = {"files": files, "seed": SEED, "runs": {}, "parse": {}}
    with tempfile.TemporaryDirectory() as root:
        write_tree(root, files)
        path = lambda n: os.path.join(root, n)          # noqa: E731
        rel = lambda p: os.path.relpath(p, root)        # noqa: E731
        P = A.AvaLabeledVideoFramePaths
        image_paths, idx_to_name, name_to_idx = P.load_image_lists(path("ava_frame_list.csv"), root)
        gold["parse"]["image_lists"] = ([[rel(p) for p in v] for v in image_paths], idx_to_name, name_to_idx)
        gold["parse"]["label_map"] = P.read_label_map(path("ava_label_map.pbtxt"))
        allowed = gold["parse"]["label_map"][1]
        for csv in ("ava_train.csv", "ava_det.csv"):
            for use_map in (False, True):
                key = (csv, use_map)
                gold["parse"][("labels",) + key] = plain(P.load_and_parse_labels_csv(
                    path(csv), name_to_idx, allowed if use_map else None))
                gold["parse"][("from_csv",) + key] = [
                    (rel(d), labels) for d, labels in P.from_csv(path("ava_frame_list.csv"), path(csv), root,
                                                                 path("ava_label_map.pbtxt") if use_map else None)]
        # each video's frames as the reference decodes them
        gold["frames"] = {}
        for name, n, _, _, _ in VIDEOS:
            v = FV.FrameVideo.from_directory(os.path.join(root, "frames", name))
            clip = get_clip(v, 0, v.duration)["video"]
            assert clip.shape[1] == n and torch.equal(clip, clip.round())
            gold["frames"][name] = clip.permute(1, 2, 3, 0).to(torch.uint8).contiguous()      # (T, H, W, 3)
        for run, (cls, args), vs, csv, use_map in RUNS:
            torch.manual_seed(SEED)
            ds = D.Ava(path("ava_frame_list.csv"), path(csv), root, path("ava_label_map.pbtxt") if use_map else None,
                       getattr(CS, cls)(*args), samplers[vs])
            log.clear()
            samples = []
            for s in ds:
                (start, end), indices = log[-1]
                want = gold["frames"][s["video_name"]][indices].permute(3, 0, 1, 2).float()
                assert torch.equal(s["video"], want), (run, s["video_name"], s["clip_index"])
                samples.append(dict({k: v for k, v in s.items() if k != "video"}, frame_indices=indices,
                                    window=(start, end)))
            windows = [(a, idx) for a, idx in log]
            gold["runs"][run] = {"sampler": (cls, args), "video_sampler": vs, "csv": csv, "label_map": use_map,
                                 "samples": samples, "get_clip_calls": windows}
    grid = []
    for dur in DURATIONS:
        s = A.TimeStampClipSampler(CS.UniformClipSampler(dur))
        for t in KEYFRAMES:
            grid.append((dur, t, tuple(s(None, 10.0, {"clip_index": t}))))
    gold["timestamp_sampler"] = grid
    torch.save(gold, GOLD)
    n = sum(len(r["samples"]) for r in gold["runs"].values())
    print("wrote %s: %d samples, %d sampler windows, %d bytes" % (GOLD, n, len(grid), os.path.getsize(GOLD)))


if __name__ == "__main__":
    main()
