"""(video path, label) pairs read from a csv file or from a directory of class directories."""
from __future__ import annotations

import os
from typing import List, Optional, Tuple

_VIDEO_EXTENSIONS = ("mp4", "avi")


class LabeledVideoPaths:
    """A list of (video path, integer label); item i is (path prefix joined with path i, {"label": label i})."""

    @classmethod
    def from_path(cls, data_path: str) -> LabeledVideoPaths:
        """``from_csv`` for a file, ``from_directory`` for a directory."""
        if os.path.isfile(data_path):
            return cls.from_csv(data_path)
        if os.path.isdir(data_path):
            return cls.from_directory(data_path)
        raise FileNotFoundError(f"{data_path} not found.")

    @classmethod
    def from_csv(cls, file_path: str) -> LabeledVideoPaths:
        """One ``<path> <integer label>`` per line, split at the last run of whitespace; a line holding only a path
        gets label -1 (an unlabelled split)."""
        assert os.path.exists(file_path), f"{file_path} not found."
        pairs = []
        with open(file_path, "r") as f:
            for line in f.read().splitlines():
                fields = line.rsplit(None, 1)
                path, label = (fields[0], -1) if len(fields) == 1 else fields
                pairs.append((path, int(label)))
        assert len(pairs) > 0, f"Failed to load dataset from {file_path}."
        return cls(pairs)

    @classmethod
    def from_directory(cls, dir_path: str) -> LabeledVideoPaths:
        """``dir_path/<class>/.../<video>.mp4|.avi``: the classes are the subdirectories, labelled 0.. in sorted
        order, and their video files are listed in sorted walk order (torchvision's ``make_dataset``)."""
        assert os.path.exists(dir_path), f"{dir_path} not found."
        classes = sorted(e.name for e in os.scandir(dir_path) if e.is_dir())
        pairs, found = [], set()
        for label, name in enumerate(classes):
            for root, _, files in sorted(os.walk(os.path.join(dir_path, name), followlinks=True)):
                for fname in sorted(files):
                    if fname.lower().endswith(_VIDEO_EXTENSIONS):
                        pairs.append((os.path.join(root, fname), label))
                        found.add(name)
        empty = sorted(set(classes) - found)
        if empty:
            raise FileNotFoundError("Found no valid file for the classes %s. Supported extensions are: %s"
                                    % (", ".join(empty), ", ".join(_VIDEO_EXTENSIONS)))
        assert len(pairs) > 0, f"Failed to load dataset from {dir_path}."
        return cls(pairs)

    def __init__(self, paths_and_labels: List[Tuple[str, Optional[int]]], path_prefix="") -> None:
        self._paths_and_labels = paths_and_labels
        self._path_prefix = path_prefix

    def _set_path_prefix(self, prefix):
        self._path_prefix = prefix

    path_prefix = property(None, _set_path_prefix, doc="Directory joined in front of every path (write-only).")

    def __getitem__(self, index: int) -> Tuple[str, dict]:
        path, label = self._paths_and_labels[index]
        return os.path.join(self._path_prefix, path), {"label": label}

    def __len__(self) -> int:
        return len(self._paths_and_labels)
