"""CPU: the AVA dataset's parsers, its keyframe clip sampler and its host-only samples against the reference's outputs
in tests/golden/ava.pt (oracle/gen_golden_ava.py), and the host side of the ragged box entry point and the detection
batch loader."""
import os
import re
from fractions import Fraction

import pytest
import torch
import torch.utils.data

from pytorchvideo_b200 import _lib
from pytorchvideo_b200 import data as D
from pytorchvideo_b200.data import clip_sampling as CS
from pytorchvideo_b200.data.ava import AvaLabeledVideoFramePaths as P
from pytorchvideo_b200.data.ava import TimeStampClipSampler
from pytorchvideo_b200.data.loader import _kept_positions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "ava.pt"), weights_only=False)
SAMPLERS = {"random": torch.utils.data.RandomSampler, "sequential": torch.utils.data.SequentialSampler}
RECORD_ONLY = ("frame_indices", "window")          # golden fields that are not sample keys


def write_fixtures(root):
    for rel, data in GOLD["files"].items():
        path = os.path.join(str(root), rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "wb") as f:
            f.write(data)
    return str(root)


def build(run, root):
    """The Ava dataset of golden run ``run``, built as oracle/gen_golden_ava.py builds the reference's."""
    r = GOLD["runs"][run]
    cls, args = r["sampler"]
    return D.Ava(os.path.join(root, "ava_frame_list.csv"), os.path.join(root, r["csv"]), root,
                 os.path.join(root, "ava_label_map.pbtxt") if r["label_map"] else None, getattr(CS, cls)(*args),
                 SAMPLERS[r["video_sampler"]])


def seeded():
    torch.manual_seed(GOLD["seed"])


def check_keys(got, want):
    assert set(got) == set(want) - set(RECORD_ONLY) | {"video"}
    for k in want:
        if k not in RECORD_ONLY:
            assert got[k] == want[k] and type(got[k]) is type(want[k]), k


# ---- parsers ---------------------------------------------------------------------------------------------------------
def test_image_lists(tmp_path):
    root = write_fixtures(tmp_path)
    paths, idx_to_name, name_to_idx = P.load_image_lists(os.path.join(root, "ava_frame_list.csv"), root)
    want = GOLD["parse"]["image_lists"]
    assert [[os.path.relpath(p, root) for p in v] for v in paths] == want[0]
    assert (idx_to_name, name_to_idx) == (want[1], want[2])
    # frames by frame_id: vidB is listed backwards, vidC has a later row from another directory
    assert want[0][1][0] == "frames/vidB/img_00001.jpg" and want[0][2][-1] == "frames/vidA/img_00001.jpg"


def test_frame_list_rows_have_five_fields(tmp_path):
    bad = tmp_path / "list.csv"
    bad.write_text("original_vido_id video_id frame_id path labels\nvidA 0 0 vidA/1.jpg\n")
    with pytest.raises(AssertionError):
        P.load_image_lists(str(bad), "")


def test_label_map(tmp_path):
    root = write_fixtures(tmp_path)
    assert P.read_label_map(os.path.join(root, "ava_label_map.pbtxt")) == GOLD["parse"]["label_map"]


@pytest.mark.parametrize("use_map", [False, True], ids=["all", "map"])
@pytest.mark.parametrize("csv", ["ava_train.csv", "ava_det.csv"])
def test_labels_csv_and_keyframes(tmp_path, csv, use_map):
    root = write_fixtures(tmp_path)
    _, _, name_to_idx = P.load_image_lists(os.path.join(root, "ava_frame_list.csv"), root)
    allowed = GOLD["parse"]["label_map"][1] if use_map else None
    got = P.load_and_parse_labels_csv(os.path.join(root, csv), name_to_idx, allowed)
    assert {v: {s: dict(d) for s, d in secs.items()} for v, secs in got.items()} == GOLD["parse"][("labels", csv, use_map)]
    paths = P.from_csv(os.path.join(root, "ava_frame_list.csv"), os.path.join(root, csv), root,
                       os.path.join(root, "ava_label_map.pbtxt") if use_map else None)
    want = GOLD["parse"][("from_csv", csv, use_map)]
    assert [(os.path.relpath(d, root), labels) for d, labels in paths] == want
    for _, labels in paths:
        assert type(labels["clip_index"]) is float and all(type(x) is float for e in labels["extra_info"] for x in e)


def test_parse_rules_in_the_golden():
    """The fixture rows exercise each rule: range, empty action, "%.2f" collisions, pruning, float seconds."""
    train = GOLD["parse"][("labels", "ava_train.csv", False)]
    assert sorted(train[0]) == [2.0, 3.0] and sorted(train[2]) == [2.0, 3.0]     # 901, 1799, 1798.5 dropped
    assert train[1][2.0]["labels"] == [1, 5, 2]                                  # "902.0" is keyframe 2.0
    assert train[0][2.0]["labels"][-1] == -1
    keyed = dict(GOLD["parse"][("from_csv", "ava_train.csv", False)][0][1])
    assert keyed["boxes"][0] == [0.1, 0.2, 0.5, 0.9] and keyed["labels"][0] == [12, 17, 80]
    mapped = GOLD["parse"][("from_csv", "ava_train.csv", True)]
    assert (0, 3.0) not in [(l["video_index"], l["clip_index"]) for _, l in mapped]   # keyframe pruned to nothing


def test_aggregate_bboxes_labels():
    got = P._aggregate_bboxes_labels({"labels": [1, 2, 3], "extra_info": [0.5, 0.25, 1.0],
                                      "boxes": [[0.1, 0.2, 0.3, 0.4], [0.3, 0.3, 0.3, 0.3], [0.104, 0.2, 0.3, 0.4]]})
    assert got == {"labels": [[1, 3], [2]], "boxes": [[0.1, 0.2, 0.3, 0.4], [0.3, 0.3, 0.3, 0.3]],
                   "extra_info": [[0.5, 1.0], [0.25]]}


def test_unknown_video_is_a_key_error(tmp_path):
    root = write_fixtures(tmp_path)
    with open(os.path.join(root, "bad.csv"), "w") as f:
        f.write("vidZ,0902,0.1,0.2,0.5,0.9,12,0\n")
    with pytest.raises(KeyError, match="vidZ"):
        D.Ava(os.path.join(root, "ava_frame_list.csv"), os.path.join(root, "bad.csv"), root,
              clip_sampler=D.UniformClipSampler(1.0))


# ---- the keyframe sampler --------------------------------------------------------------------------------------------
def test_timestamp_sampler_windows():
    for dur, t, want in GOLD["timestamp_sampler"]:
        got = TimeStampClipSampler(D.UniformClipSampler(dur))(None, 10.0, {"clip_index": t})
        assert repr(tuple(got)) == repr(want), (dur, t)
        assert type(got) is D.ClipInfo


def test_timestamp_sampler_takes_any_clip_duration():
    class Fixed:
        _clip_duration = Fraction(3, 4)

    s = TimeStampClipSampler(Fixed())
    assert tuple(s(0.0, 1.0, {"clip_index": 2.0})) == (1.625, 2.375, 0, 0, True)
    s = TimeStampClipSampler(D.RandomClipSampler(0.5))
    assert tuple(s(None, None, {"clip_index": 2.0})) == (1.75, 2.25, 0, 0, True)
    s.reset()


# ---- host-only samples -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("run", sorted(GOLD["runs"]))
def test_host_only_samples_equal_the_reference(tmp_path, run):
    root = write_fixtures(tmp_path)
    seeded()
    got = list(build(run, root).host_only())
    want = GOLD["runs"][run]["samples"]
    assert len(got) == len(want)
    for g, w in zip(got, want):
        check_keys(g, w)
        clip = g["video"]
        assert isinstance(clip, D.ClipFrames)
        assert clip.frame_indices == w["frame_indices"] and clip.kept == list(range(len(w["frame_indices"])))
        folder = os.path.join(root, "frames", w["video_name"])
        names = sorted(os.listdir(folder), key=lambda n: [int(p) if p.isdigit() else p for p in re.split(r"(\d+)", n)])
        assert clip.paths == [os.path.join(folder, names[i]) for i in w["frame_indices"]]
        for path, blob in zip(clip.paths, clip.data):
            with open(path, "rb") as f:
                assert f.read() == blob


def test_window_before_zero_is_skipped():
    runs = GOLD["runs"]
    assert any(idx is None and a[0] < 0 for a, idx in runs["random"]["get_clip_calls"])
    assert all(s["clip_index"] == 3.0 for s in runs["random"]["samples"])


def test_host_only_keeps_the_transforms_frames(tmp_path):
    root = write_fixtures(tmp_path)
    ds = build("uniform", root).host_only(keep=lambda n: _kept_positions(4, n))
    s = next(iter(ds))
    assert s["video"].kept == _kept_positions(4, len(s["video"].frame_indices)) and len(s["video"].paths) == 4


# ---- the ragged box entry point and the loader, host side ------------------------------------------------------------
def test_header_declares_the_ragged_box_entry_point():
    hdr = open(os.path.join(ROOT, "include", "pv_b200.h")).read()
    assert ("int pv_clip_boxes_transform_ragged(const pv_boxes_desc* d, const void* boxes_in, const int32_t* box_start,"
            "\n                                   const int32_t* geom, const int32_t* geom_host,"
            "\n                                   void* boxes_out, float* rois_out, void* stream);") in hdr
    assert re.search(r"#define PV_BOX_DENORM 64\b", hdr) and re.search(r"#define PV_BOX_ALL_STEPS 63\b", hdr)
    assert _lib.BOX_DENORM == 64 and "pv_clip_boxes_transform_ragged" in _lib.SIGNATURES


def test_existing_entry_point_rejects_denorm():
    """PV_BOX_DENORM is not a step of pv_clip_boxes_transform: its host check refuses it before any launch."""
    import ctypes
    d = _lib.BoxesDesc()
    d.n_clips, d.n_boxes, d.steps, d.dtype, d.out_h, d.out_w = 1, 0, _lib.BOX_DENORM, _lib.BOX_F32, 8, 8
    assert _lib.load().pv_clip_boxes_transform(ctypes.byref(d), None, None, None, None, None, None) == -1
    assert "unknown step bits 0x40" in _lib.last_error()


def test_ragged_entry_point_host_checks():
    import ctypes
    lib = _lib.load()
    d = _lib.BoxesDesc()
    d.n_clips, d.n_boxes, d.steps, d.dtype, d.out_h, d.out_w = 1, 0, 127, _lib.BOX_F64, 8, 8
    rows = (ctypes.c_int32 * 7)(20, 30, 20, 30, 0, 0, 1)
    call = lambda: lib.pv_clip_boxes_transform_ragged(ctypes.byref(d), None, None, rows, rows, None, None, None)  # noqa
    assert call() == 0                                     # no boxes: validated, nothing launched
    d.steps = 128
    assert call() == -1 and "unknown step bits" in _lib.last_error()
    d.steps = 127
    rows[4] = 13
    assert call() == -1 and "window" in _lib.last_error()


def test_detection_loader_rejects_what_it_cannot_run(tmp_path):
    from pytorchvideo_b200.transforms import FusedClipTransform, FusedDetectionTransform
    root = write_fixtures(tmp_path)
    with pytest.raises(TypeError, match="FusedDetectionTransform"):
        D.DetectionBatchLoader(build("uniform", root), 2, FusedClipTransform(4))
    tr = FusedDetectionTransform(4, (0.45,) * 3, (0.225,) * 3, short_side=16)
    with pytest.raises(ValueError, match="box_dtype"):
        D.DetectionBatchLoader(build("uniform", root), 2, tr, box_dtype=torch.float16)
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="DetectionBatchLoader .*no CPU path"):
            next(iter(D.DetectionBatchLoader(build("uniform", root), 2, tr)))
