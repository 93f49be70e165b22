"""ClipBatchLoader: batches of a frame-video dataset as network input, with one decode and one transform launch."""
import functools

import torch
import torch.utils.data

from .. import _lib as L
from ..transforms import FusedClipTransform
from ..transforms import functional as Fv
from .jpeg import decode_batch


def _kept_positions(num_samples, n_frames):
    """The positions FusedClipTransform keeps of an n_frames clip: its temporal subsample, drawing nothing."""
    if num_samples is None:
        return list(range(n_frames))
    return Fv.temporal_indices(n_frames, num_samples).tolist()


def _collate(samples):
    return samples


class ClipBatchLoader:
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
        self.dataset = dataset.host_only(keep=functools.partial(_kept_positions, transform.num_samples))
        self.transform = transform
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
            raise RuntimeError("ClipBatchLoader decodes and transforms on the GPU and has no CPU path")
        L.require_device()
        for samples in self._host_batches():
            yield self.collate(samples)

    def collate(self, samples):
        """One batch from the host-only samples (dicts whose "video" is a ClipFrames record)."""
        for s in samples:
            if isinstance(s["video"], list):
                raise NotImplementedError("ClipBatchLoader takes one clip per sample; multi-clip samplers give "
                                          "lists of clips")
        paths, data, where = unique_frames([s["video"] for s in samples])
        flat, sizes = decode_batch(data, out_dtype=torch.uint8, names=paths)
        starts = [0]
        for h, w in sizes:
            starts.append(starts[-1] + 3 * h * w)
        offs, geom = [], []
        for s, pos in zip(samples, where):
            hw = {sizes[u] for u in pos}
            if len(hw) > 1:
                odd = next(paths[u] for u in pos if sizes[u] != sizes[pos[0]])
                raise RuntimeError("video %s: frame %s is %dx%d, the clip's first frame %dx%d: the frames of a clip "
                                   "must share one size" % (s.get("video_name"), odd, sizes[paths.index(odd)][1],
                                                            sizes[paths.index(odd)][0], sizes[pos[0]][1],
                                                            sizes[pos[0]][0]))
            H, W = sizes[pos[0]]
            idx, resize, win, flip = self.transform.plan((3, len(s["video"].frame_indices), H, W))
            nh, nw = (H, W) if resize is None else resize
            geom.append(((H, W), (nh, nw), (0, 0, nh, nw) if win is None else win, flip))
            offs.append([starts[u] for u in pos])
        out_hws = {g[2][2:] for g in geom}
        if len(out_hws) > 1:
            raise RuntimeError("the clips of a batch come out at different sizes %s; give the transform a crop"
                               % sorted(out_hws))
        if len({len(o) for o in offs}) > 1:
            raise RuntimeError("the clips of a batch keep different frame counts; give the transform num_samples")
        t = self.transform
        video = Fv.clip_transform_ragged(flat, offs, geom, out_hws.pop(), mean=t.mean, std=t.std, div255=t.div255,
                                         out_dtype=t.out_dtype, slow_alpha=t.slowfast_alpha)
        batch = {"video": video}
        for key in samples[0]:
            if key != "video":
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
