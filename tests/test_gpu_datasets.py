"""GPU: the datasets' decoded clips against the reference's (tests/golden/datasets.pt), the ragged mode of the batched
clip kernel against a float64 restatement and against per-clip launches, and ClipBatchLoader against the per-sample
chain (dataset sample -> FusedClipTransform)."""
import os

import numpy as np
import pytest
import torch

from pytorchvideo_b200 import _lib as L
from pytorchvideo_b200 import data as D
from pytorchvideo_b200.transforms import FusedClipTransform
from pytorchvideo_b200.transforms import functional as Fv
from test_datasets import GOLD, build, seeded, write_fixtures

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
MEAN, STD = (0.45, 0.43, 0.40), (0.225, 0.22, 0.23)


@pytest.mark.parametrize("name", sorted(GOLD["runs0"]))
def test_dataset_clips_equal_the_reference(tmp_path, name):
    root = write_fixtures(tmp_path)
    run = GOLD["runs0"][name]
    seeded()
    got = list(build(name, root, run["sampler"]))
    assert len(got) == len(run["samples"])
    for g, w in zip(got, run["samples"]):
        assert g["video"].is_cuda and g["video"].dtype == torch.float32
        assert torch.equal(g["video"].cpu(), w["video"].float())
        assert {k: v for k, v in g.items() if k != "video"} == {k: v for k, v in w.items()
                                                                if k not in ("video", "frame_indices")}


# ---- ragged launches against float64 -----------------------------------------------------------------------------------
def ref_clip(frames, geom, out_hw, mean, std, div255):
    """float64 restatement of one clip: /255, normalise, ATen's bilinear taps (fp32 index arithmetic), crop, flip."""
    (ih, iw), (nh, nw), (top, left, oh, ow), flip = geom
    y0, y1, ly = Fv.bilinear_table(ih, nh)
    x0, x1, lx = Fv.bilinear_table(iw, nw)
    ys = slice(top, top + oh)
    xs = np.arange(left, left + ow)[::-1] if flip else np.arange(left, left + ow)
    out = []
    for f in frames:
        v = f.astype(np.float64)
        if div255:
            v = v / 255.0
        if mean is not None:
            v = (v - np.array(mean)) / np.array(std)
        a, b, l1 = y0[ys], y1[ys], ly[ys].astype(np.float64)[:, None, None]
        c, d, m1 = x0[xs], x1[xs], lx[xs].astype(np.float64)[None, :, None]
        r0 = v[a][:, c] * (1 - m1) + v[a][:, d] * m1
        r1 = v[b][:, c] * (1 - m1) + v[b][:, d] * m1
        out.append((r0 * (1 - l1) + r1 * l1).transpose(2, 0, 1))
    return np.stack(out, 1)          # (3, n_t, oh, ow)


def ragged_case(sizes, n_t, out_hw, seed, src_dtype, scale=1.0, far=False, flip=False, repeat=False):
    """Random frames of the given per-clip sizes packed as decode_batch packs them, and one geometry per clip."""
    rng = np.random.default_rng(seed)
    blobs, offs, frames, geom = [], [], [], []
    pos = 0
    for b, (h, w) in enumerate(sizes):
        n_src = max(1, n_t // 2) if repeat else n_t
        clip = [rng.integers(0, 256, (h, w, 3)).astype(np.uint8) for _ in range(n_src)]
        starts = []
        for f in clip:
            blobs.append(f.reshape(-1))
            starts.append(pos)
            pos += f.size
        pick = sorted(rng.integers(0, n_src, n_t).tolist()) if repeat else list(range(n_t))
        offs.append([starts[k] for k in pick])
        frames.append([clip[k] for k in pick])
        oh, ow = out_hw
        nh, nw = max(oh, int(round(h * scale))), max(ow, int(round(w * scale)))
        top, left = ((nh - oh, nw - ow) if far else (int(rng.integers(0, nh - oh + 1)), int(rng.integers(0, nw - ow + 1))))
        geom.append(((h, w), (nh, nw), (top, left, oh, ow), bool(flip and b % 2 == 0)))
    src = torch.from_numpy(np.concatenate(blobs))
    if src_dtype == torch.float32:
        src = src.float()
    return src.to(DEV), offs, frames, geom


CASES = {
    # name: (sizes, n_t, out_hw, scale, far, flip, repeat, slow_alpha)
    "1x1": ([(1, 1), (1, 1)], 3, (1, 1), 1.0, False, False, False, None),
    "1xN_up": ([(1, 9), (1, 5)], 2, (4, 7), 3.0, False, True, False, None),
    "Nx1_up": ([(9, 1), (6, 1)], 2, (5, 3), 2.5, True, False, False, None),
    "down_far_flip": ([(91, 67), (40, 77), (64, 64)], 4, (17, 23), 0.4, True, True, False, None),
    "up_mixed": ([(23, 31), (30, 40), (17, 45)], 5, (33, 41), 2.2, False, True, False, None),
    "slow": ([(23, 31), (17, 45)], 8, (16, 16), 1.0, False, True, False, 4),
    "one_clip": ([(37, 29)], 6, (20, 20), 1.0, True, False, False, 2),
    "repeats": ([(26, 26), (30, 40)], 8, (24, 24), 1.3, False, True, True, 4),
    "b64": ([(16 + (b * 7) % 23, 16 + (b * 11) % 29) for b in range(64)], 4, (16, 16), 1.0, False, True, False, None),
}


@pytest.mark.parametrize("src_dtype", [torch.uint8, torch.float32], ids=["u8", "f32"])
@pytest.mark.parametrize("out_dtype", [torch.float16, torch.float32], ids=["f16", "f32"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_ragged_against_float64(case, src_dtype, out_dtype):
    sizes, n_t, out_hw, scale, far, flip, repeat, alpha = CASES[case]
    src, offs, frames, geom = ragged_case(sizes, n_t, out_hw, 7, src_dtype, scale, far, flip, repeat)
    got = Fv.clip_transform_ragged(src, offs, geom, out_hw, mean=MEAN, std=STD, div255=True, out_dtype=out_dtype,
                                   slow_alpha=alpha)
    fast = got[1] if alpha else got
    want = np.stack([ref_clip(f, g, out_hw, MEAN, STD, True) for f, g in zip(frames, geom)])
    tol = 2e-2 if out_dtype == torch.float16 else 2e-5
    np.testing.assert_allclose(fast.float().cpu().numpy(), want, rtol=tol, atol=tol)
    if alpha:
        sidx = Fv.slow_pathway_indices(n_t, alpha)
        assert torch.equal(got[0], fast[:, :, sidx])


@pytest.mark.parametrize("out_dtype", [torch.float16, torch.float32], ids=["f16", "f32"])
def test_ragged_equals_per_clip_batch_launches(out_dtype):
    sizes, n_t, out_hw = [(23, 31), (30, 40), (17, 45), (64, 48)], 6, (16, 16)
    src, offs, frames, geom = ragged_case(sizes, n_t, out_hw, 3, torch.uint8, 1.4, False, True, True)
    got = Fv.clip_transform_ragged(src, offs, geom, out_hw, mean=MEAN, std=STD, div255=True, out_dtype=out_dtype,
                                   slow_alpha=2)
    for b, (f, g) in enumerate(zip(frames, geom)):
        clip = torch.from_numpy(np.stack(f)).to(DEV).permute(3, 0, 1, 2)      # (3, T, H, W), THWC strides
        want = Fv.clip_transform_batch(clip, resize_hw=g[1], window=g[2], hflip=g[3], mean=MEAN, std=STD, div255=True,
                                       out_dtype=out_dtype, slow_alpha=2)
        assert torch.equal(got[0][b], want[0]) and torch.equal(got[1][b], want[1]), b


def test_ragged_host_checks():
    src, offs, frames, geom = ragged_case([(20, 20)], 2, (8, 8), 1, torch.uint8)
    lib = L.load()
    with pytest.raises(RuntimeError, match="GPU only"):
        Fv.clip_transform_ragged(src.cpu(), offs, geom, (8, 8))
    with pytest.raises(RuntimeError, match="outside the source buffer"):
        Fv.clip_transform_ragged(src[:100], offs, geom, (8, 8))
    # the entry point's own checks, called directly
    import ctypes as C
    offs_d = torch.tensor(offs, dtype=torch.int64, device=DEV).view(-1)
    d = L.ClipBatchDesc()
    d.C, d.n_clips, d.n_t, d.out_h, d.out_w, d.src_dtype, d.dst_dtype = 3, 1, 2, 8, 8, L.PV_U8, L.PV_F32
    out = torch.empty((1, 3, 2, 8, 8), device=DEV)
    d.d_clip = out.stride(0)

    def call(rows, **kw):
        for k, v in kw.items():
            setattr(d, k, v)
        host = torch.tensor(rows, dtype=torch.int32)
        dev = host.to(DEV)
        return lib.pv_clip_transform_ragged(C.byref(d), src.data_ptr(), offs_d.data_ptr(), dev.data_ptr(),
                                            host.data_ptr(), None, out.data_ptr(), None,
                                            torch.cuda.current_stream().cuda_stream)

    assert call([20, 20, 20, 20, 0, 0, 0]) == 0
    torch.cuda.synchronize()
    assert call([20, 20, 20, 20, 13, 0, 0]) == -1 and "window" in L.last_error()
    assert call([20, 20, 20, 20, 0, -1, 0]) == -1
    assert call([1 << 15, 1 << 15, 20, 20, 0, 0, 0]) == -1 and "32-bit" in L.last_error()
    assert call([20, 20, 20, 20, 0, 0, 0], C=4) == -1 and "3 channels" in L.last_error()
    assert call([20, 20, 20, 20, 0, 0, 0], C=3, n_clips=0) == -1 and "empty" in L.last_error()


# ---- the batch loader --------------------------------------------------------------------------------------------------
def per_sample_batches(ds, transform, batch_size):
    """The per-sample chain: each normal-mode sample through ``transform``, stacked per batch."""
    out, cur = [], []
    for s in ds:
        cur.append((transform(s["video"]), s))
        if len(cur) == batch_size:
            out.append(cur)
            cur = []
    if cur:
        out.append(cur)
    return out


def stack(items, slowfast):
    if slowfast:
        return [torch.stack([v[0] for v, _ in items]), torch.stack([v[1] for v, _ in items])]
    return torch.stack([v for v, _ in items])


@pytest.mark.parametrize("slowfast", [True, False], ids=["slowfast", "single"])
def test_loader_equals_the_per_sample_chain(tmp_path, slowfast):
    root = write_fixtures(tmp_path)
    tr = FusedClipTransform(8 if slowfast else 4, MEAN, STD, random_short_side=(18, 30), crop=("random", 16),
                            hflip_prob=0.5, slowfast_alpha=4 if slowfast else None, out_dtype=torch.float16)
    seeded()
    want = per_sample_batches(build("labeled_uniform_backpad", root, "sequential"), tr, 3)
    seeded()
    got = list(D.ClipBatchLoader(build("labeled_uniform_backpad", root, "sequential"), 3, tr))
    assert len(got) == len(want) and len(want) > 2
    for g, w in zip(got, want):
        exp = stack(w, slowfast)
        if slowfast:
            assert torch.equal(g["video"][0], exp[0]) and torch.equal(g["video"][1], exp[1])
        else:
            assert torch.equal(g["video"], exp)
        for key in ("label", "video_name", "video_index", "clip_index", "aug_index"):
            assert g[key] == [s[key] for _, s in w]


def test_loader_in_workers_equals_the_in_process_loader(tmp_path):
    root = write_fixtures(tmp_path)
    tr = FusedClipTransform(8, MEAN, STD, short_side=20, crop=("center", 16), slowfast_alpha=4)

    def clips(num_workers):       # {(video, clip): (slow, fast)}: the workers interleave their batches
        loader = D.ClipBatchLoader(build("charades_uniform", root, "sequential"), 2, tr, num_workers=num_workers)
        return {key: (x["video"][0][k], x["video"][1][k]) for x in loader
                for k, key in enumerate(zip(x["video_index"], x["clip_index"]))}

    clips_a, clips_b = clips(0), clips(2)
    assert clips_a.keys() == clips_b.keys()
    for k in clips_a:
        assert torch.equal(clips_a[k][0], clips_b[k][0]) and torch.equal(clips_a[k][1], clips_b[k][1])


def test_loader_launches_one_decode_and_one_transform(tmp_path):
    root = write_fixtures(tmp_path)
    tr = FusedClipTransform(8, MEAN, STD, short_side=20, crop=("center", 16), slowfast_alpha=4)
    it = iter(D.ClipBatchLoader(build("labeled_uniform_backpad", root, "sequential"), 4, tr))
    next(it)                                       # first batch loads the library and the modules
    before = L.kernel_counts()
    batch = next(it)
    torch.cuda.synchronize()
    after = L.kernel_counts()
    delta = {k: v - before.get(k, 0) for k, v in after.items() if v != before.get(k, 0)}
    assert delta.pop("jpeg_huffman_kernel") == 1 and delta.pop("jpeg_idct_islow_kernel") == 1
    colour = {k: delta.pop(k) for k in list(delta) if k.startswith("jpeg_ycc_rgb_kernel<")}
    assert colour and all(v == 1 and k.endswith(",u8>") for k, v in colour.items())
    assert delta == {"clip_transform_batch_kernel<uint8_t,__half,3,true>": 1}, delta
    assert batch["video"][1].shape[0] == len(batch["label"])


def test_loader_dedups_repeated_frames(tmp_path):
    root = write_fixtures(tmp_path)
    # 8 kept of a 4-frame clip: each frame file repeats, and is decoded once
    tr = FusedClipTransform(8, MEAN, STD, short_side=20, crop=("center", 16))
    loader = D.ClipBatchLoader(build("charades_uniform", root, "sequential"), 2, tr)
    samples = [next(iter(loader.dataset))]
    paths, _, where = D.loader.unique_frames([s["video"] for s in samples])
    assert len(paths) == 4 and len(where[0]) == 8
    batch = loader.collate(samples)
    assert batch["video"].shape == (1, 3, 8, 16, 16)


def test_loader_errors(tmp_path):
    root = write_fixtures(tmp_path)
    tr = FusedClipTransform(4, MEAN, STD, short_side=20, crop=("center", 16))
    # a frame of another size inside one clip
    odd = os.path.join(root, "frames", "vid1", "frame_2.jpg")
    with open(os.path.join(root, "frames", "vid0", "frame_1.jpg"), "rb") as f:
        other = f.read()
    with open(odd, "wb") as f:
        f.write(other)
    ds = build("charades_uniform", root, "sequential")
    with pytest.raises(RuntimeError, match=r"video 1: frame .*vid1/frame_2\.jpg is 31x23"):
        list(D.ClipBatchLoader(ds, 4, tr))
    # a corrupt frame is named by its path
    root2 = write_fixtures(tmp_path / "b")
    bad = os.path.join(root2, "frames", "vid0", "frame_1.jpg")
    with open(bad, "rb") as f:
        blob = f.read()
    with open(bad, "wb") as f:
        f.write(blob[:len(blob) // 3])
    with pytest.raises(RuntimeError, match=r"vid0/frame_1\.jpg: "):
        list(D.ClipBatchLoader(build("charades_uniform", root2, "sequential"), 4, tr))
    # multi-clip samples
    kin = os.path.join(root2, "kinetics.csv")
    ds = D.Kinetics(kin, D.RandomMultiClipSampler(0.2, 2), torch.utils.data.SequentialSampler, video_path_prefix=root2,
                    decode_audio=False)
    with pytest.raises(NotImplementedError, match="multi-clip"):
        list(D.ClipBatchLoader(ds, 2, tr))
