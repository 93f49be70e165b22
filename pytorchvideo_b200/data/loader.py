"""Batch loaders: batches of a frame-video dataset as network input, with one decode and one transform launch.

``ClipBatchLoader`` batches clips; ``DetectionBatchLoader`` batches clips with their boxes and the RoI rows of the
detection heads."""
import functools

import torch
import torch.utils.data

from .. import _lib as L
from ..transforms import FusedClipTransform, FusedDetectionTransform
from ..transforms import functional as Fv
from .jpeg import decode_batch


def _kept_positions(num_samples, n_frames):
    """The positions FusedClipTransform keeps of an n_frames clip: its temporal subsample, drawing nothing."""
    if num_samples is None:
        return list(range(n_frames))
    return Fv.temporal_indices(n_frames, num_samples).tolist()


def _collate(samples):
    return samples


class _FrameBatchLoader:
    """What the loaders share: host-only samples read in DataLoader workers, batched, and decoded by one
    ``decode_batch`` in this process."""

    def __init__(self, dataset, batch_size, num_samples, num_workers, drop_last):
        self.dataset = dataset.host_only(keep=functools.partial(_kept_positions, num_samples))
        self.batch_size, self.num_workers, self.drop_last = batch_size, num_workers, drop_last

    def _host_batches(self):
        if self.num_workers > 0:
            yield from torch.utils.data.DataLoader(self.dataset, batch_size=self.batch_size,
                                                   num_workers=self.num_workers, drop_last=self.drop_last,
                                                   collate_fn=_collate)
            return
        # in this process without a DataLoader, whose iterator draws a worker seed from torch's global RNG: the only
        # global draws between samples are then the dataset's and the transform's, as in a per-sample loop
        batch = []
        for sample in self.dataset:
            batch.append(sample)
            if len(batch) == self.batch_size:
                yield batch
                batch = []
        if batch and not self.drop_last:
            yield batch

    def __iter__(self):
        if not torch.cuda.is_available():
            raise RuntimeError("%s decodes and transforms on the GPU and has no CPU path" % type(self).__name__)
        L.require_device()
        for samples in self._host_batches():
            yield self.collate(samples)

    def _decode(self, samples):
        """One decode_batch of the samples' distinct frame files: (their paths, the packed uint8 frames, each frame's
        (h, w), each frame's element offset, per sample the distinct-frame index of each kept frame)."""
        for s in samples:
            if isinstance(s["video"], list):
                raise NotImplementedError("%s takes one clip per sample; multi-clip samplers give lists of clips"
                                          % type(self).__name__)
        paths, data, where = unique_frames([s["video"] for s in samples])
        flat, sizes = decode_batch(data, out_dtype=torch.uint8, names=paths)
        starts = [0]
        for h, w in sizes:
            starts.append(starts[-1] + 3 * h * w)
        return paths, flat, sizes, starts, where

    @staticmethod
    def _clip_size(sample, pos, paths, sizes):
        """The (H, W) the kept frames ``pos`` of ``sample`` share."""
        hw = {sizes[u] for u in pos}
        if len(hw) > 1:
            odd = next(paths[u] for u in pos if sizes[u] != sizes[pos[0]])
            raise RuntimeError("video %s: frame %s is %dx%d, the clip's first frame %dx%d: the frames of a clip "
                               "must share one size" % (sample.get("video_name"), odd, sizes[paths.index(odd)][1],
                                                        sizes[paths.index(odd)][0], sizes[pos[0]][1],
                                                        sizes[pos[0]][0]))
        return sizes[pos[0]]

    @staticmethod
    def _out_size(geom, offs):
        """The one output (h, w) of the batch's windows, which must also keep one frame count."""
        out_hws = {g[2][2:] for g in geom}
        if len(out_hws) > 1:
            raise RuntimeError("the clips of a batch come out at different sizes %s; give the transform a crop"
                               % sorted(out_hws))
        if len({len(o) for o in offs}) > 1:
            raise RuntimeError("the clips of a batch keep different frame counts; give the transform num_samples")
        return out_hws.pop()


class ClipBatchLoader(_FrameBatchLoader):
    """Iterates ``dataset`` in batches of ``batch_size`` clips transformed by ``transform``, on the current GPU.

    The dataset is switched to its host-only mode: DataLoader workers (``num_workers``; 0 reads in this process) read
    only the files of the frames ``transform`` keeps.  Then each batch takes, in this process:
      1. one ``decode_batch`` of the batch's distinct frame files, as uint8, at their own sizes (its host parse gives
         the frame sizes the plans need);
      2. ``transform.plan`` per sample, in sample order: the global-RNG draws of calling ``transform`` on each sample;
      3. one ``pv_clip_transform_ragged`` launch into (B, 3, n_t, h, w), or [slow, fast] with ``slowfast_alpha``.
    The batch is {"video": that tensor, and every other key of the samples: the list of their values in order}.  It
    equals stacking ``transform(sample["video"])`` over the dataset's normal-mode samples under the same seeds.

    ``transform`` is a FusedClipTransform without random_resized_crop.  Clips of one batch may differ in size, but
    the frames of one clip may not, and the transform must give every clip the same output size and frame count.
    """

    def __init__(self, dataset, batch_size, transform, num_workers=0, drop_last=False):
        if not isinstance(transform, FusedClipTransform):
            raise TypeError("transform must be a FusedClipTransform")
        if transform.random_resized_crop is not None:
            raise NotImplementedError("random_resized_crop has no ragged-batch kernel")
        super().__init__(dataset, batch_size, transform.num_samples, num_workers, drop_last)
        self.transform = transform

    def collate(self, samples):
        """One batch from the host-only samples (dicts whose "video" is a ClipFrames record)."""
        paths, flat, sizes, starts, where = self._decode(samples)
        offs, geom = [], []
        for s, pos in zip(samples, where):
            H, W = self._clip_size(s, pos, paths, sizes)
            idx, resize, win, flip = self.transform.plan((3, len(s["video"].frame_indices), H, W))
            nh, nw = (H, W) if resize is None else resize
            geom.append(((H, W), (nh, nw), (0, 0, nh, nw) if win is None else win, flip))
            offs.append([starts[u] for u in pos])
        out_hw = self._out_size(geom, offs)
        t = self.transform
        video = Fv.clip_transform_ragged(flat, offs, geom, out_hw, mean=t.mean, std=t.std, div255=t.div255,
                                         out_dtype=t.out_dtype, slow_alpha=t.slowfast_alpha)
        batch = {"video": video}
        for key in samples[0]:
            if key != "video":
                batch[key] = [s[key] for s in samples]
        return batch


class DetectionBatchLoader(_FrameBatchLoader):
    """Iterates a detection dataset (e.g. ``Ava``) in batches of ``batch_size`` clips with their boxes, transformed by
    the FusedDetectionTransform ``transform``, on the current GPU.

    Workers read the host-only samples as for ``ClipBatchLoader``.  Then each batch takes, in this process:
      1. one ``decode_batch`` of the batch's distinct frame files;
      2. ``transform.plan`` per sample, in sample order (the torch and numpy draws of a per-sample loop);
      3. one copy of the geometry rows {in_h, in_w, new_h, new_w, top, left, hflip}, the frame offsets and the box
         offsets to the device, and one of the boxes;
      4. one ``pv_clip_transform_ragged`` launch: (B, 3, n_t, h, w), or [slow, fast] with ``slowfast_alpha``;
      5. one ``pv_clip_boxes_transform_ragged`` launch on the same geometry rows.
    The batch is {"video", "boxes": per clip a (K_b, 4) view of one transformed ``box_dtype`` tensor, "rois": the fp32
    (K, 5) rows (batch position, x1, y1, x2, y2) for ``model(video, rois)``, and every other key of the samples: the
    list of their values}.  The samples' ``boxes_key`` holds (K_b, 4) boxes, in [0, 1] when ``normalized_boxes`` is
    set (AVA's), else in source pixels.

    Exactness: under the same torch and numpy seeds a batch is ``torch.equal`` to this per-sample chain on the
    dataset's normal-mode samples: ``b = torch.tensor(sample[boxes_key], dtype=box_dtype)``, times
    ``torch.tensor([W, H, W, H], dtype=box_dtype)`` of the clip's frame size when ``normalized_boxes`` is set; then
    ``video, rois = transform(sample["video"], b)``; the videos stacked, the RoI rows concatenated with column 0 set
    to the clip's batch position, and each clip's boxes equal to its RoI columns 1..4 in ``box_dtype`` (the same box
    steps with ``FusedDetectionTransform``'s rounding).  Clips of one batch may differ in size; the transform must
    give them one output size (a crop, or a fixed short side on one aspect ratio).
    """

    def __init__(self, dataset, batch_size, transform, num_workers=0, drop_last=False, boxes_key="boxes",
                 normalized_boxes=True, box_dtype=torch.float32):
        if not isinstance(transform, FusedDetectionTransform):
            raise TypeError("transform must be a FusedDetectionTransform")
        if box_dtype not in (torch.float32, torch.float64):
            raise ValueError("box_dtype must be torch.float32 or torch.float64")
        super().__init__(dataset, batch_size, transform.num_samples, num_workers, drop_last)
        self.transform = transform
        self.boxes_key, self.normalized_boxes, self.box_dtype = boxes_key, normalized_boxes, box_dtype

    def collate(self, samples):
        """One batch from the host-only samples (dicts whose "video" is a ClipFrames record)."""
        for s in samples:
            if self.boxes_key not in s:
                raise KeyError("sample of video %s has no %r boxes" % (s.get("video_name"), self.boxes_key))
        paths, flat, sizes, starts, where = self._decode(samples)
        offs, geom, boxes, box_start = [], [], [], [0]
        for s, pos in zip(samples, where):
            H, W = self._clip_size(s, pos, paths, sizes)
            resize, win, flip = self.transform.plan((3, len(s["video"].frame_indices), H, W))
            geom.append(((H, W), resize, win, flip))
            offs.append([starts[u] for u in pos])
            b = torch.tensor(s[self.boxes_key], dtype=self.box_dtype).reshape(-1, 4)
            boxes.append(b)
            box_start.append(box_start[-1] + b.shape[0])
        out_hw = self._out_size(geom, offs)
        frame_off, rows = Fv.ragged_tables(offs, geom, out_hw)
        # one host-to-device copy: the int64 frame offsets, then the int32 geometry rows and box offsets
        B, n_off, n_rows = len(samples), frame_off.numel(), rows.numel()
        host = torch.zeros(n_off + (n_rows + B + 2) // 2, dtype=torch.int64)
        host[:n_off] = frame_off
        tail = host[n_off:].view(torch.int32)
        tail[:n_rows] = rows
        tail[n_rows:n_rows + B + 1] = torch.tensor(box_start, dtype=torch.int32)
        tables = host.to(flat.device)
        offs_d = tables[:n_off]
        rows_d = tables[n_off:].view(torch.int32)[:n_rows]
        start_d = tables[n_off:].view(torch.int32)[n_rows:n_rows + B + 1]
        t = self.transform
        video = Fv.launch_clip_ragged(flat, offs_d, rows_d, rows, B, out_hw, mean=t.mean, std=t.std,
                                      div255=t.div255, out_dtype=t.out_dtype, slow_alpha=t.slowfast_alpha)
        steps = t.box_steps() | (L.BOX_DENORM if self.normalized_boxes else 0)
        boxes_d = torch.cat(boxes).to(flat.device)
        out, rois = Fv.clip_boxes_transform_ragged(boxes_d, steps, start_d, rows_d, rows, out_hw, rois=True)
        rois._pv_keepalive = (boxes_d, tables)
        batch = {"video": video, "boxes": [out[s:e] for s, e in zip(box_start[:-1], box_start[1:])], "rois": rois}
        for key in samples[0]:
            if key not in ("video", self.boxes_key):
                batch[key] = [s[key] for s in samples]
        return batch


def unique_frames(clips):
    """The distinct frame files of a batch of ClipFrames: (paths, their bytes, per clip the distinct-frame index of
    each kept frame)."""
    index, paths, data, where = {}, [], [], []
    for clip in clips:
        pos = []
        for path, blob in zip(clip.paths, clip.data):
            if path not in index:
                index[path] = len(paths)
                paths.append(path)
                data.append(blob)
            pos.append(index[path])
        where.append(pos)
    return paths, data, where
