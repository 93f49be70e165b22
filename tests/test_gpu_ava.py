"""GPU: the AVA dataset's decoded clips against the reference's (tests/golden/ava.pt), the ragged box entry point
(pv_clip_boxes_transform_ragged) against per-clip launches, the torch DENORM expression and a float64 restatement,
and DetectionBatchLoader against the per-sample chain (dataset sample -> boxes to pixels -> FusedDetectionTransform),
down to a detection model's output."""
import numpy as np
import pytest
import torch

from pytorchvideo_b200 import _lib as L
from pytorchvideo_b200 import data as D
from pytorchvideo_b200 import testing as TS
from pytorchvideo_b200.transforms import FusedDetectionTransform
from pytorchvideo_b200.transforms import functional as Fv
from test_ava import GOLD, build, check_keys, seeded, write_fixtures

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
MEAN, STD = (0.45, 0.43, 0.40), (0.225, 0.22, 0.23)
BITS = {torch.float32: torch.int32, torch.float64: torch.int64}


@pytest.mark.parametrize("run", sorted(GOLD["runs"]))
def test_dataset_clips_equal_the_reference(tmp_path, run):
    root = write_fixtures(tmp_path)
    seeded()
    got = list(build(run, root))
    want = GOLD["runs"][run]["samples"]
    assert len(got) == len(want)
    for g, w in zip(got, want):
        check_keys(g, w)
        assert g["video"].is_cuda and g["video"].dtype == torch.float32
        clip = GOLD["frames"][w["video_name"]][w["frame_indices"]].permute(3, 0, 1, 2).float()
        assert torch.equal(g["video"].cpu(), clip)


# ---- the ragged box kernel -------------------------------------------------------------------------------------------
SIZES = [(23, 31), (33, 21), (19, 27), (240, 320), (256, 340)]     # (H, W): landscape, portrait, odd, AVA-like
OUT_HW = (16, 16)


def ragged_geom(sizes, seed):
    """Per clip ((H, W), (new_h, new_w), (top, left, out_h, out_w), hflip) with a random short side and crop."""
    rng = np.random.default_rng(seed)
    geom = []
    for b, (h, w) in enumerate(sizes):
        nh, nw = Fv.short_side_size(h, w, int(rng.integers(16, 40)))
        top, left = int(rng.integers(0, nh - OUT_HW[0] + 1)), int(rng.integers(0, nw - OUT_HW[1] + 1))
        geom.append(((h, w), (nh, nw), (top, left) + OUT_HW, b % 2 == 0))
    return geom


def ragged_boxes(counts, sizes, dtype, normalized, seed):
    """(K, 4) boxes per clip: random ones reaching past the frame, and the edge rows - NaN, signed zeros, the frame
    edges, values far outside."""
    rng = np.random.default_rng(seed)
    out = []
    for n, (h, w) in zip(counts, sizes):
        sx, sy = (1.0, 1.0) if normalized else (float(w), float(h))
        b = np.stack([rng.uniform(-0.1, 1.1, n) * sx, rng.uniform(-0.1, 1.1, n) * sy,
                      rng.uniform(-0.1, 1.1, n) * sx, rng.uniform(-0.1, 1.1, n) * sy], 1)
        edges = [[np.nan, 0.5 * sy, sx, np.nan], [-0.0, -0.0, 0.0, 0.0], [0.0, 0.0, sx, sy],
                 [sx - (0 if normalized else 1), sy - (0 if normalized else 1), sx, sy], [-40.0, -1e-30, 1e6, 5e3],
                 [1 / 3 * sx, 2 / 3 * sy, 0.7 * sx, 0.9 * sy]]
        if n:
            b[:min(n, len(edges))] = edges[:n]
        out.append(torch.from_numpy(b).to(dtype))
    return out


def launch_ragged(boxes, geom, steps, rois=True):
    offs = [[0]] * len(geom)
    _, rows = Fv.ragged_tables(offs, geom, OUT_HW)
    start = [0] + np.cumsum([b.shape[0] for b in boxes]).tolist()
    start_d = torch.tensor(start, dtype=torch.int32, device=DEV)
    flat = torch.cat(boxes).to(DEV)
    out, r = Fv.clip_boxes_transform_ragged(flat, steps, start_d, rows.to(DEV), rows, OUT_HW, rois=rois)
    return out, r, start


def per_clip(boxes, geom, steps):
    """pv_clip_boxes_transform on each clip by itself: (boxes, rois) per clip."""
    res = []
    for b, ((h, w), nhw, (top, left, _, _), flip) in zip(boxes, geom):
        res.append(Fv.clip_boxes_transform(b.to(DEV).contiguous(), steps, in_hw=(h, w), new_hw=nhw, offset=(top, left),
                                           hflip=flip, out_hw=OUT_HW, rois=True))
    return res


def same_bits(a, b):
    """Bit-equal, signed zeros included; a NaN matches a NaN (the GPU's multiply returns its canonical NaN, the CPU's
    keeps the operand's payload)."""
    a, b = a.cpu().contiguous(), b.cpu().contiguous()
    if a.shape != b.shape or a.dtype != b.dtype or not torch.equal(torch.isnan(a), torch.isnan(b)):
        return False
    a, b = a.masked_fill(torch.isnan(a), 0.0), b.masked_fill(torch.isnan(b), 0.0)
    return torch.equal(a.view(BITS[a.dtype]), b.view(BITS[b.dtype]))


def torch_denorm(boxes, sizes):
    return [b * torch.tensor([w, h, w, h], dtype=b.dtype) for b, (h, w) in zip(boxes, sizes)]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_ragged_equals_per_clip_launches_for_every_step_subset(dtype):
    counts = [7, 0, 9, 1, 12]
    geom = ragged_geom(SIZES, 3)
    pix = ragged_boxes(counts, SIZES, dtype, False, 5)
    unit = ragged_boxes(counts, SIZES, dtype, True, 6)
    denormed = torch_denorm(unit, SIZES)
    for steps in range(64):
        for src, extra, ref_src in ((pix, 0, pix), (unit, L.BOX_DENORM, denormed)):
            out, rois, start = launch_ragged(src, geom, steps | extra)
            for b, (want, want_rois) in enumerate(per_clip(ref_src, geom, steps)):
                s, e = start[b], start[b + 1]
                assert same_bits(out[s:e], want), (steps, extra, b)
                assert same_bits(rois[s:e, 1:], want_rois[:, 1:]), (steps, extra, b)
                assert torch.equal(rois[s:e, 0], torch.full((e - s,), float(b), device=DEV)), (steps, b)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_denorm_is_the_torch_expression(dtype):
    counts = [5, 3, 0, 8, 6]
    unit = ragged_boxes(counts, SIZES, dtype, True, 11)
    out, _, start = launch_ragged(unit, ragged_geom(SIZES, 4), L.BOX_DENORM, rois=False)
    want = torch.cat(torch_denorm(unit, SIZES))
    assert same_bits(out.cpu(), want)
    assert torch.isnan(out[start[0]]).tolist() == [True, False, False, True]      # NaN passes through


def ref64(boxes, geom, steps):
    """The box chain in float64 numpy, one clip: DENORM, clip to the source, scale, crop, clip, flip, clip."""
    (h, w), (nh, nw), (top, left, oh, ow), flip = geom
    b = boxes.astype(np.float64).copy()
    clip = lambda v, hi: np.minimum(float(hi), np.maximum(0.0, v))     # noqa: E731
    if steps & L.BOX_DENORM:
        b = b * np.array([w, h, w, h], np.float64)
    if steps & L.BOX_CLIP_SRC:
        b[:, 0::2], b[:, 1::2] = clip(b[:, 0::2], w - 1), clip(b[:, 1::2], h - 1)
    if steps & L.BOX_SCALE:
        b = b * (nh / h if w < h else nw / w)
    if steps & L.BOX_CROP:
        b[:, 0::2], b[:, 1::2] = b[:, 0::2] - left, b[:, 1::2] - top
    for bit in (L.BOX_CLIP_CROP, L.BOX_FLIP, L.BOX_CLIP_OUT):
        if steps & bit and bit != L.BOX_FLIP:
            b[:, 0::2], b[:, 1::2] = clip(b[:, 0::2], ow - 1), clip(b[:, 1::2], oh - 1)
        elif steps & bit and flip:
            b[:, 0], b[:, 2] = (ow - b[:, 2]) - 1, (ow - b[:, 0]) - 1
    return b


@pytest.mark.parametrize("steps", [127, 64 | 1 | 2 | 32, 2 | 4 | 16, 63], ids=lambda s: "steps%d" % s)
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_ragged_against_float64(dtype, steps):
    counts = [4, 6, 0, 9, 3]
    geom = ragged_geom(SIZES, 8)
    boxes = ragged_boxes(counts, SIZES, dtype, bool(steps & L.BOX_DENORM), 9)
    out, rois, start = launch_ragged(boxes, geom, steps)
    out, rois = out.cpu().double().numpy(), rois.cpu().numpy()
    for b, (bx, g) in enumerate(zip(boxes, geom)):
        want = ref64(bx.numpy(), g, steps)
        got = out[start[b]:start[b + 1]]
        assert np.array_equal(np.isnan(got), np.isnan(want))
        if dtype == torch.float64:             # one rounding per operation in float64: the restatement itself
            np.testing.assert_array_equal(got + 0.0, want + 0.0)
        else:                                  # a few float32 roundings of coordinates below 2^10
            np.testing.assert_allclose(got, want, rtol=5e-7, atol=2e-4)
        np.testing.assert_array_equal(rois[start[b]:start[b + 1], 1:], got.astype(np.float32))
        clipped = want[~np.isnan(want).any(1)]
        if steps & L.BOX_CLIP_OUT and clipped.size:
            assert clipped[:, 0::2].max() <= OUT_HW[1] - 1 and clipped.min() >= 0


def test_ragged_zero_boxes_and_empty_clips():
    geom = ragged_geom(SIZES[:3], 1)
    boxes = [torch.zeros((0, 4)), torch.tensor([[0.0, 0.0, 1.0, 1.0]]), torch.zeros((0, 4))]
    (out, rois, start), ran = TS.launched_kernels(launch_ragged, boxes, geom, 127)
    assert ran == {"clip_boxes_ragged_kernel<float>": 1}
    assert start == [0, 0, 1, 1] and rois[:, 0].tolist() == [1.0]
    none = [torch.zeros((0, 4), dtype=torch.float64)] * 3
    (out, rois, _), ran = TS.launched_kernels(launch_ragged, none, geom, 127)
    assert ran == {} and out.shape == (0, 4) and rois.shape == (0, 5)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_ragged_ledger(dtype):
    geom = ragged_geom(SIZES, 2)
    boxes = ragged_boxes([3, 2, 1, 4, 5], SIZES, dtype, True, 2)
    _, ran = TS.launched_kernels(launch_ragged, boxes, geom, 127)
    assert ran == {"clip_boxes_ragged_kernel<%s>" % ("float" if dtype == torch.float32 else "double"): 1}


def test_ragged_geom_host_checks():
    geom = ragged_geom(SIZES[:2], 1)
    _, rows = Fv.ragged_tables([[0]] * 2, geom, OUT_HW)
    flat = torch.rand(3, 4, device=DEV)
    start = torch.tensor([0, 1, 3], dtype=torch.int32, device=DEV)
    rows_d = rows.to(DEV)

    def call(host, steps=127, out_hw=OUT_HW):
        return Fv.clip_boxes_transform_ragged(flat, steps, start, rows_d, host, out_hw)

    call(rows)
    for field, value, msg in ((0, 0, "bad frame size"), (3, 0, "bad frame size"), (4, 40, "window"),
                              (12, -1, "window")):
        bad = rows.clone()
        bad[field] = value
        with pytest.raises(RuntimeError, match=msg):
            call(bad)
    with pytest.raises(RuntimeError, match="unknown step bits 0x80"):
        call(rows, steps=128)
    with pytest.raises(RuntimeError, match="bad output frame"):
        call(rows, out_hw=(0, 16))
    with pytest.raises(RuntimeError, match="7 ints per clip"):
        call(rows[:10])
    # the existing entry point keeps refusing the new bit
    with pytest.raises(RuntimeError, match="unknown step bits 0x40"):
        Fv.clip_boxes_transform(flat, L.BOX_DENORM, in_hw=(20, 20), out_hw=OUT_HW)


# ---- the loader ------------------------------------------------------------------------------------------------------
def seed_all(s=7):
    torch.manual_seed(s)
    np.random.seed(s)


def per_sample_batches(ds, transform, batch_size, box_dtype):
    """The per-sample chain: normal-mode sample, boxes to pixels in torch, FusedDetectionTransform; per batch."""
    out, cur = [], []
    for s in ds:
        H, W = s["video"].shape[-2:]
        b = torch.tensor(s["boxes"], dtype=box_dtype) * torch.tensor([W, H, W, H], dtype=box_dtype)
        cur.append((transform(s["video"], b), s))
        if len(cur) == batch_size:
            out.append(cur)
            cur = []
    if cur:
        out.append(cur)
    return out


def check_batch(got, items, slowfast):
    vids = [v for (v, _), _ in items]
    if slowfast:
        assert torch.equal(got["video"][0], torch.stack([v[0] for v in vids]))
        assert torch.equal(got["video"][1], torch.stack([v[1] for v in vids]))
    else:
        assert torch.equal(got["video"], torch.stack(vids))
    rois = []
    for pos, ((_, r), _) in enumerate(items):
        r = r.clone()
        r[:, 0] = pos
        rois.append(r)
    assert torch.equal(got["rois"], torch.cat(rois))
    for b, ((_, r), _) in enumerate(items):
        assert torch.equal(got["boxes"][b].float(), r[:, 1:])
    for key in ("labels", "extra_info", "video_index", "clip_index", "aug_index", "video_name"):
        assert got[key] == [s[key] for _, s in items]


LOADER_CASES = {
    # name: (slowfast, crop, box dtype, run)
    "slowfast_random_f32": (True, "random", torch.float32, "uniform"),
    "single_uniform_f32": (False, "uniform", torch.float32, "uniform_map"),
    "slowfast_uniform_f64": (True, "uniform", torch.float64, "random"),
    "single_random_f64": (False, "random", torch.float64, "uniform"),
}


def detection_transform(slowfast, crop, out_dtype=torch.float16):
    if crop == "random":
        return FusedDetectionTransform(8 if slowfast else 4, MEAN, STD, random_short_side=(18, 30),
                                       crop=("random", 16), hflip_prob=0.5, slowfast_alpha=4 if slowfast else None,
                                       out_dtype=out_dtype)
    return FusedDetectionTransform(8 if slowfast else 4, MEAN, STD, short_side=20, crop=("uniform", 16, 1),
                                   slowfast_alpha=4 if slowfast else None, out_dtype=out_dtype)


@pytest.mark.parametrize("case", sorted(LOADER_CASES))
def test_loader_equals_the_per_sample_chain(tmp_path, case):
    slowfast, crop, box_dtype, run = LOADER_CASES[case]
    root = write_fixtures(tmp_path)
    tr = detection_transform(slowfast, crop)
    seed_all()
    want = per_sample_batches(build(run, root), tr, 2, box_dtype)
    seed_all()
    got = list(D.DetectionBatchLoader(build(run, root), 2, tr, box_dtype=box_dtype))
    assert len(got) == len(want) and len(want) >= 2
    for g, w in zip(got, want):
        assert all(b.dtype == box_dtype for b in g["boxes"])
        check_batch(g, w, slowfast)


def test_loader_in_workers_equals_the_in_process_loader(tmp_path):
    root = write_fixtures(tmp_path)
    tr = detection_transform(True, "uniform")

    def batches(num_workers):       # {(video, keyframe): (slow, fast, boxes, rois)}: the workers interleave batches
        loader = D.DetectionBatchLoader(build("uniform", root), 2, tr, num_workers=num_workers)
        out = {}
        for x in loader:
            for k, key in enumerate(zip(x["video_index"], x["clip_index"])):
                rows = x["rois"][x["rois"][:, 0] == k, 1:]
                out[key] = (x["video"][0][k], x["video"][1][k], x["boxes"][k], rows)
        return out

    a, b = batches(0), batches(8)
    assert a.keys() == b.keys() and len(a) == len(GOLD["runs"]["uniform"]["samples"])
    for k in a:
        assert all(torch.equal(x, y) for x, y in zip(a[k], b[k])), k


def test_loader_launches_one_decode_one_clip_and_one_box_kernel(tmp_path):
    root = write_fixtures(tmp_path)
    tr = detection_transform(True, "random")
    it = iter(D.DetectionBatchLoader(build("uniform", root), 3, tr))
    next(it)                                       # the first batch loads the library and the modules
    batch, delta = TS.launched_kernels(next, it)
    torch.cuda.synchronize()
    assert delta.pop("jpeg_huffman_kernel") == 1 and delta.pop("jpeg_idct_islow_kernel") == 1
    colour = {k: delta.pop(k) for k in list(delta) if k.startswith("jpeg_ycc_rgb_kernel<")}
    assert colour and all(v == 1 and k.endswith(",u8>") for k, v in colour.items())
    assert delta == {"clip_transform_batch_kernel<uint8_t,__half,3,true>": 1, "clip_boxes_ragged_kernel<float>": 1}, delta
    assert batch["video"][1].shape[0] == 3 and batch["rois"].shape[0] == sum(b.shape[0] for b in batch["boxes"])


def test_loader_errors(tmp_path):
    root = write_fixtures(tmp_path)
    # a short side without a crop on mixed aspect ratios: the clips come out at different sizes
    tr = FusedDetectionTransform(4, MEAN, STD, short_side=20)
    with pytest.raises(RuntimeError, match="come out at different sizes"):
        list(D.DetectionBatchLoader(build("uniform", root), 3, tr))
    tr = detection_transform(False, "uniform")
    with pytest.raises(KeyError, match="gt_boxes"):
        list(D.DetectionBatchLoader(build("uniform", root), 2, tr, boxes_key="gt_boxes"))
    loader = D.DetectionBatchLoader(build("uniform", root), 2, tr)
    sample = next(iter(loader.dataset))
    with pytest.raises(NotImplementedError, match="multi-clip"):
        loader.collate([dict(sample, video=[sample["video"], sample["video"]])])
    with pytest.raises(TypeError):
        D.DetectionBatchLoader(build("uniform", root), 2, None)


def test_detection_model_on_a_loader_batch(tmp_path):
    import pytorchvideo_b200.models.hub as PH
    root = write_fixtures(tmp_path)
    tr = FusedDetectionTransform(4, MEAN, STD, random_short_side=(64, 72), crop=("random", 64), hflip_prob=0.5,
                                 out_dtype=torch.float32)
    seed_all(3)
    want = per_sample_batches(build("uniform", root), tr, 3, torch.float32)[0]
    seed_all(3)
    got = next(iter(D.DetectionBatchLoader(build("uniform", root), 3, tr)))
    check_batch(got, want, False)
    model = TS.randomize_model(PH.slow_r50_detection(head_activation=None), seed=1234, f16_weights=True).eval().cuda()
    try:
        rois = []
        for pos, ((_, r), _) in enumerate(want):
            r = r.clone()
            r[:, 0] = pos
            rois.append(r)
        ref = model(torch.stack([v for (v, _), _ in want]), torch.cat(rois)).float().cpu()
        out = model(got["video"], got["rois"]).float().cpu()
    finally:
        model.cpu()
    assert out.shape == (got["rois"].shape[0], ref.shape[1]) and torch.isfinite(out).all()
    assert torch.equal(out, ref)
