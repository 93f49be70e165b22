"""CPU: clip samplers, the frame-folder datasets in their host-only mode, and the batch loader's host side, against the
reference's outputs in tests/golden/datasets.pt (oracle/gen_golden_datasets.py)."""
import logging
import os
import random
from fractions import Fraction

import pytest
import torch
import torch.utils.data

from pytorchvideo_b200 import _lib
from pytorchvideo_b200 import data as D
from pytorchvideo_b200.data import clip_sampling as CS
from pytorchvideo_b200.data.loader import _kept_positions, unique_frames
from pytorchvideo_b200.transforms import functional as Fv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "datasets.pt"), weights_only=False)
SAMPLERS = {"random": torch.utils.data.RandomSampler, "sequential": torch.utils.data.SequentialSampler}


def write_fixtures(root):
    for rel, data in GOLD["files"].items():
        path = os.path.join(root, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "wb") as f:
            f.write(data)
    return str(root)


def build(name, root, sampler):
    """The dataset of golden run ``name``, built as oracle/gen_golden_datasets.py builds the reference's."""
    root = str(root)
    vs = SAMPLERS[sampler]
    csv = os.path.join(root, "charades.csv")
    ssv2 = [os.path.join(root, n) for n in ("ssv2_labels.json", "ssv2_train.json", "ssv2.csv")]
    kin = os.path.join(root, "kinetics.csv")
    return {
        "charades_uniform": lambda: D.Charades(csv, D.UniformClipSampler(Fraction(1, 5)), vs, video_path_prefix=root,
                                               frames_per_clip=4),
        "charades_constant": lambda: D.Charades(csv, D.ConstantClipsPerVideoSampler(0.1, 2, 2), vs,
                                                video_path_prefix=root),
        "ssv2_random": lambda: D.SSv2(*ssv2, D.RandomClipSampler(0.2), vs, video_path_prefix=root, frames_per_clip=5,
                                      rand_sample_frames=True),
        "ssv2_middle": lambda: D.SSv2(*ssv2, D.UniformClipSampler(0.2), vs, video_path_prefix=root, frames_per_clip=3),
        "kinetics_random": lambda: D.Kinetics(kin, D.RandomClipSampler(0.25), vs, video_path_prefix=root,
                                              decode_audio=False),
        "labeled_uniform_backpad": lambda: D.labeled_video_dataset(kin, D.UniformClipSampler(Fraction(4, 30), None, True),
                                                                   vs, video_path_prefix=root, decode_audio=False),
        "kinetics_decode_audio_default": lambda: D.Kinetics(kin, D.RandomClipSampler(0.25), vs, video_path_prefix=root),
    }[name]()


def seeded():
    torch.manual_seed(GOLD["seed"])
    random.seed(GOLD["seed"])


def check_sample(got, want, with_indices):
    """A host-only sample against the reference's: same keys, same values, the same frames."""
    assert set(got) == set(want) - {"frame_indices"}
    for k in want:
        if k not in ("video", "frame_indices"):
            assert got[k] == want[k] and type(got[k]) is type(want[k]), k
    clip = got["video"]
    assert isinstance(clip, D.ClipFrames)
    assert clip.kept == list(range(want["video"].shape[1])) and len(clip.data) == len(clip.paths) == len(clip.kept)
    if with_indices:
        assert clip.frame_indices == want["frame_indices"]
    for path, blob in zip(clip.paths, clip.data):
        with open(path, "rb") as f:
            assert f.read() == blob


# ---- clip samplers ---------------------------------------------------------------------------------------------------
def test_samplers_equal_the_reference():
    keys = []
    for entry in GOLD["samplers"]:
        if entry[0] not in keys:
            keys.append(entry[0])
    for (cls, args), dur, first, want in GOLD["samplers"]:
        random.seed(keys.index((cls, args)))
        s = getattr(CS, cls)(*args)
        last, got = first, []
        for _ in range(40):
            c = s(last, dur, {})
            got.append(tuple(c))
            last = c.clip_end_sec
            if c.is_last_clip[-1] if isinstance(c.is_last_clip, list) else c.is_last_clip:
                break
        assert repr(got) == repr(want), (cls, args, dur, first)


def test_make_clip_sampler():
    for kind, args, name in GOLD["make_clip_sampler"]:
        assert type(D.make_clip_sampler(kind, *args)).__name__ == name
    with pytest.raises(NotImplementedError):
        D.make_clip_sampler("nearest", 1.0)


# ---- paths -----------------------------------------------------------------------------------------------------------
def test_labeled_video_paths(tmp_path):
    root = write_fixtures(tmp_path)
    lp = D.LabeledVideoPaths.from_path(os.path.join(root, "classes"))
    assert [(os.path.relpath(lp[i][0], root), lp[i][1]) for i in range(len(lp))] == GOLD["class_directory"]
    lp = D.LabeledVideoPaths.from_path(os.path.join(root, "kinetics.csv"))
    assert [lp[i] for i in range(len(lp))] == GOLD["csv_paths"]
    lp.path_prefix = "/data"
    assert lp[0] == ("/data/frames/vid0", {"label": 3})
    with pytest.raises(FileNotFoundError):
        D.LabeledVideoPaths.from_path(os.path.join(root, "absent"))


# ---- datasets, host-only ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(GOLD["runs0"]))
def test_host_only_sequence_equals_the_reference(tmp_path, name):
    root = write_fixtures(tmp_path)
    run = GOLD["runs0"][name]
    ds = build(name, root, run["sampler"]).host_only()
    seeded()
    got = list(ds)
    assert len(got) == len(run["samples"])
    for g, w in zip(got, run["samples"]):
        check_sample(g, w, True)


@pytest.mark.parametrize("name", sorted(GOLD["runs2"]))
def test_host_only_sequence_in_two_workers(tmp_path, name):
    root = write_fixtures(tmp_path)
    run = GOLD["runs2"][name]
    ds = build(name, root, run["sampler"]).host_only()
    seeded()
    got = list(torch.utils.data.DataLoader(ds, batch_size=None, num_workers=2))
    assert len(got) == len(run["samples"])
    for g, w in zip(got, run["samples"]):
        check_sample(g, w, False)


def test_host_only_keep_reads_only_the_kept_frames(tmp_path):
    root = write_fixtures(tmp_path)
    ds = build("ssv2_middle", root, "sequential").host_only(keep=lambda n: [0, n - 1, n - 1])
    s = next(iter(ds))
    clip = s["video"]
    assert clip.kept == [0, 2, 2] and len(clip.frame_indices) == 3
    assert clip.paths[1] == clip.paths[2] and clip.data[1] is clip.data[2]


def test_video_file_is_a_logged_load_failure(tmp_path, caplog):
    root = write_fixtures(tmp_path)
    with open(os.path.join(root, "bad.csv"), "w") as f:
        f.write("clips/bad.mp4 0\n" * 12)
    ds = D.labeled_video_dataset(os.path.join(root, "bad.csv"), D.RandomClipSampler(0.2),
                                 torch.utils.data.SequentialSampler, video_path_prefix=root, decode_audio=False)
    with caplog.at_level(logging.ERROR):
        with pytest.raises(RuntimeError, match="Failed to load video after 10 retries"):
            next(iter(ds.host_only()))
    text = "\n".join(r.exc_text or "" for r in caplog.records) + "\n".join(
        str(r.exc_info[1]) for r in caplog.records if r.exc_info)
    assert "NotImplementedError" in text and "bad.mp4" in text and "no video-file decoder" in text


def test_normal_mode_refuses_a_worker(tmp_path):
    root = write_fixtures(tmp_path)
    ds = build("charades_uniform", root, "sequential")
    with pytest.raises(RuntimeError, match="ClipBatchLoader"):
        list(torch.utils.data.DataLoader(ds, batch_size=None, num_workers=1))


def test_multi_process_sampler_splits_in_runs():
    class Info:
        def __init__(self, i):
            self.id, self.num_workers = i, 3

    import pytorchvideo_b200.data.utils as U
    real = U.torch.utils.data.get_worker_info
    got = []
    try:
        for i in range(3):
            U.torch.utils.data.get_worker_info = lambda i=i: Info(i)
            got.append(list(D.MultiProcessSampler(torch.utils.data.SequentialSampler(range(7)))))
    finally:
        U.torch.utils.data.get_worker_info = real
    assert got == [[0, 1, 2], [3, 4], [5, 6]]


# ---- loader, host side -----------------------------------------------------------------------------------------------
def test_unique_frames_dedup():
    a = D.ClipFrames([b"x", b"y", b"y"], ["/a/1", "/a/2", "/a/2"], [0, 1], [0, 1, 1])
    b = D.ClipFrames([b"y", b"z"], ["/a/2", "/b/1"], [1, 5], [0, 1])
    paths, data, where = unique_frames([a, b])
    assert paths == ["/a/1", "/a/2", "/b/1"] and data == [b"x", b"y", b"z"]
    assert where == [[0, 1, 1], [1, 2]]


def test_kept_positions_are_the_transforms():
    assert _kept_positions(None, 5) == [0, 1, 2, 3, 4]
    assert _kept_positions(4, 10) == Fv.temporal_indices(10, 4).tolist()
    assert _kept_positions(8, 3) == Fv.temporal_indices(3, 8).tolist() == [0, 0, 0, 0, 1, 1, 1, 2]


def test_ragged_tables():
    offs, rows = Fv.ragged_tables([[0, 300], [300, 300]], [((10, 10), (12, 12), (1, 2, 8, 8), True),
                                                           ((5, 20), (8, 32), (0, 24, 8, 8), False)], (8, 8))
    assert offs.tolist() == [0, 300, 300, 300] and offs.dtype == torch.int64
    assert rows.tolist() == [10, 10, 12, 12, 1, 2, 1, 5, 20, 8, 32, 0, 24, 0] and rows.dtype == torch.int32
    with pytest.raises(RuntimeError, match="crop window"):
        Fv.ragged_tables([[0]], [((10, 10), (10, 10), (0, 0, 9, 9), False)], (8, 8))
    with pytest.raises(RuntimeError, match="one entry per clip"):
        Fv.ragged_tables([[0], [0]], [((10, 10), (10, 10), (0, 0, 8, 8), False)], (8, 8))


def test_loader_rejects_what_it_cannot_run(tmp_path):
    from pytorchvideo_b200.transforms import FusedClipTransform
    root = write_fixtures(tmp_path)
    rrc = FusedClipTransform(4, random_resized_crop={"target_height": 8, "target_width": 8, "scale": (0.5, 1.0),
                                                     "aspect_ratio": (0.75, 1.33)})
    with pytest.raises(NotImplementedError):
        D.ClipBatchLoader(build("charades_uniform", root, "sequential"), 2, rrc)
    if not torch.cuda.is_available():
        loader = D.ClipBatchLoader(build("charades_uniform", root, "sequential"), 2, FusedClipTransform(4))
        with pytest.raises(RuntimeError, match="no CPU path"):
            next(iter(loader))


def test_ragged_entry_point_is_bound():
    assert "pv_clip_transform_ragged" in _lib.SIGNATURES
