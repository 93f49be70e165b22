"""AVA Actions stored as image frames: the keyframe annotations, their boxes, and the clip around each keyframe."""
from __future__ import annotations

import os
from collections import defaultdict
from typing import Any, Callable, Dict, Optional, Set, Tuple, Type

import torch
import torch.utils.data

from .clip_sampling import ClipInfo, ClipSampler
from .labeled_video_dataset import LabeledVideoDataset


class AvaLabeledVideoFramePaths:
    """Parses the AVA csv files (frame lists, keyframe labels, label map) into ``(video frame directory, labels)``
    pairs, one per annotated keyframe (`<https://research.google.com/ava/download.html>`_)."""

    # keyframe seconds that carry annotations, and where the annotated part of a video starts
    AVA_VALID_FRAMES = list(range(902, 1799))
    FPS = 30
    AVA_VIDEO_START_SEC = 900

    @classmethod
    def _aggregate_bboxes_labels(cls, inp: Dict):
        """One entry per distinct box (keyed by its "%.2f" coordinates; the first box of a key keeps its coordinates),
        with the list of its labels and of its extra infos."""
        labels, extra_info, boxes = inp["labels"], inp["extra_info"], inp["boxes"]
        labels_agg, extra_info_agg, boxes_agg = [], [], []
        bb_dict = {}
        for i in range(len(labels)):
            bbox_key = "{:.2f},{:.2f},{:.2f},{:.2f}".format(boxes[i][0], boxes[i][1], boxes[i][2], boxes[i][3])
            if bbox_key not in bb_dict:
                bb_dict[bbox_key] = len(boxes_agg)
                boxes_agg.append(boxes[i])
                labels_agg.append([])
                extra_info_agg.append([])
            idx = bb_dict[bbox_key]
            labels_agg[idx].append(labels[i])
            extra_info_agg[idx].append(extra_info[i])
        return {"labels": labels_agg, "boxes": boxes_agg, "extra_info": extra_info_agg}

    @classmethod
    def from_csv(cls, frame_paths_file: str, frame_labels_file: str, video_path_prefix: str,
                 label_map_file: Optional[str] = None):
        """
        Args:
            frame_paths_file: space-separated file with a header line, then one
                ``<original_vido_id video_id frame_id rel_path labels>`` row per frame.
            frame_labels_file: csv of ``<video_id, keyframe_sec, x1, y1, x2, y2, action_label, detection_iou>`` or
                ``<..., action_label, person_id>`` rows; boxes in [0, 1].
            video_path_prefix: prefix of every ``rel_path``.
            label_map_file: .pbtxt of class ids and names; when given, labels outside it are dropped.
        Returns:
            a list of ``(video frame directory, {"labels", "boxes", "extra_info", "video_index", "clip_index"})``, one
            per keyframe that keeps a label.
        """
        allowed_class_ids = None
        if label_map_file is not None:
            _, allowed_class_ids = AvaLabeledVideoFramePaths.read_label_map(label_map_file)
        image_paths, _, video_name_to_idx = AvaLabeledVideoFramePaths.load_image_lists(frame_paths_file,
                                                                                       video_path_prefix)
        video_frame_labels = AvaLabeledVideoFramePaths.load_and_parse_labels_csv(frame_labels_file, video_name_to_idx,
                                                                                 allowed_class_ids)
        labeled_video_paths = []
        for video_id in video_frame_labels.keys():
            for frame_video_sec in video_frame_labels[video_id].keys():
                labels = video_frame_labels[video_id][frame_video_sec]
                if len(labels["labels"]) > 0:
                    labels = AvaLabeledVideoFramePaths._aggregate_bboxes_labels(labels)
                    labels["video_index"] = video_id
                    labels["clip_index"] = frame_video_sec
                    # the clip is read from every file of the directory of the video's first listed frame
                    labeled_video_paths.append((os.path.dirname(image_paths[video_id][0]), labels))
        return labeled_video_paths

    @staticmethod
    def load_and_parse_labels_csv(frame_labels_file: str, video_name_to_idx: dict,
                                  allowed_class_ids: Optional[Set] = None):
        """{video index: {keyframe second - 900: {"boxes": [[x1, y1, x2, y2]], "labels": [int], "extra_info":
        [float]}}} of the rows whose second lies in [902, 1798].  An empty label is -1; a label outside
        ``allowed_class_ids`` (when given) drops its row; a video missing from ``video_name_to_idx`` is a KeyError."""
        labels_dict = {}
        with open(frame_labels_file, "r") as f:
            for line in f:
                row = line.strip().split(",")
                video_idx = video_name_to_idx[row[0]]
                frame_sec = float(row[1])
                if (frame_sec > AvaLabeledVideoFramePaths.AVA_VALID_FRAMES[-1]
                        or frame_sec < AvaLabeledVideoFramePaths.AVA_VALID_FRAMES[0]):
                    continue
                # the frames of a video start at second 900
                frame_sec = frame_sec - AvaLabeledVideoFramePaths.AVA_VIDEO_START_SEC
                bbox = list(map(float, row[2:6]))
                label = -1 if row[6] == "" else int(row[6])
                if (allowed_class_ids is not None) and (label not in allowed_class_ids):
                    continue
                extra_info = float(row[7])           # detection iou or person id, both as float
                if video_idx not in labels_dict:
                    labels_dict[video_idx] = {}
                if frame_sec not in labels_dict[video_idx]:
                    labels_dict[video_idx][frame_sec] = defaultdict(list)
                labels_dict[video_idx][frame_sec]["boxes"].append(bbox)
                labels_dict[video_idx][frame_sec]["labels"].append(label)
                labels_dict[video_idx][frame_sec]["extra_info"].append(extra_info)
        return labels_dict

    @staticmethod
    def load_image_lists(frame_paths_file: str, video_path_prefix: str) -> Tuple:
        """(frame paths per video in frame_id order, video names by index, {video name: index}), videos in first-seen
        order.  The header line is skipped and every row must have 5 fields."""
        image_paths, video_name_to_idx, video_idx_to_name = [], {}, []
        with open(frame_paths_file, "r") as f:
            f.readline()
            for line in f:
                row = line.split()
                assert len(row) == 5
                video_name = row[0]
                if video_name not in video_name_to_idx:
                    video_name_to_idx[video_name] = len(video_name_to_idx)
                    video_idx_to_name.append(video_name)
                    image_paths.append({})
                image_paths[video_name_to_idx[video_name]][int(row[2])] = os.path.join(video_path_prefix, row[3])
        image_paths_list = [[paths[key] for key in sorted(paths)] for paths in image_paths]
        return image_paths_list, video_idx_to_name, video_name_to_idx

    @staticmethod
    def read_label_map(label_map_file: str) -> Tuple:
        """({class id: name}, {class ids}) of a .pbtxt: ids from ``  id:`` or ``  label_id:`` lines, each named by the
        last ``  name:`` line before it."""
        label_map, class_ids = {}, set()
        name = ""
        with open(label_map_file, "r") as f:
            for line in f:
                if line.startswith("  name:"):
                    name = line.split('"')[1]
                elif line.startswith("  id:") or line.startswith("  label_id:"):
                    class_id = int(line.strip().split(" ")[-1])
                    label_map[class_id] = name
                    class_ids.add(class_id)
        return label_map, class_ids


class TimeStampClipSampler:
    """The clip centred on an annotation's keyframe: [t - d / 2, t - d / 2 + d) for the ``_clip_duration`` d of
    ``clip_sampler``, always clip 0, augmentation 0 and the video's last clip (each keyframe reloads its video)."""

    def __init__(self, clip_sampler: ClipSampler) -> None:
        self.clip_sampler = clip_sampler

    def __call__(self, last_clip_time: float, video_duration: float, annotation: Dict[str, Any]) -> ClipInfo:
        """``last_clip_time`` and ``video_duration`` are not used; ``annotation["clip_index"]`` is the keyframe
        second."""
        center_frame_sec = annotation["clip_index"]
        clip_start_sec = center_frame_sec - self.clip_sampler._clip_duration / 2.0
        return ClipInfo(clip_start_sec, clip_start_sec + self.clip_sampler._clip_duration, 0, 0, True)

    def reset(self) -> None:
        pass


def Ava(frame_paths_file: str, frame_labels_file: str, video_path_prefix: str = "",
        label_map_file: Optional[str] = None, clip_sampler: Callable = ClipSampler,
        video_sampler: Type[torch.utils.data.Sampler] = torch.utils.data.RandomSampler,
        transform: Optional[Callable[[dict], Any]] = None) -> LabeledVideoDataset:
    """AVA keyframes as a ``LabeledVideoDataset`` of frame-folder videos (30 fps, no audio).

    A sample is the clip ``TimeStampClipSampler(clip_sampler)`` centres on a keyframe, with "boxes" (in [0, 1]),
    "labels", "extra_info", "video_index" (the frame list's video index), "clip_index" (the keyframe second, counted
    from 900 s), "aug_index" and "video_name".  A keyframe whose window starts before 0 s has no clip and is skipped.
    Arguments as ``AvaLabeledVideoFramePaths.from_csv`` and ``LabeledVideoDataset``; ``transform`` sees the clip and
    its boxes.  ``host_only()`` yields file bytes instead (see ``DetectionBatchLoader``).
    """
    labeled_video_paths = AvaLabeledVideoFramePaths.from_csv(frame_paths_file, frame_labels_file, video_path_prefix,
                                                             label_map_file)
    return LabeledVideoDataset(labeled_video_paths=labeled_video_paths, clip_sampler=TimeStampClipSampler(clip_sampler),
                               transform=transform, video_sampler=video_sampler, decode_audio=False)
