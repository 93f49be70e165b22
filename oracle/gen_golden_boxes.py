"""Golden vectors of the detection input transforms (tests/golden/boxes.pt).

Runs the reference's box-aware functions (transforms/functional.py:195-445) on the CPU for every case of
pytorchvideo_b200.testing.BOX_FUNCTIONAL_CASES, on float32 and float64 boxes, under fixed torch and numpy seeds.  For
every case it asserts that the reference's boxes are reproduced bit for bit by the arithmetic the box kernel states
(one rounding to the boxes' dtype per operation: scale by T(new / old), subtract the offset, numpy's clip, the flip
as (W - x2) - 1).  It stores the output boxes and the draws read back from the reference's outputs (the side from the
scaled clip, the crop offsets from the view's storage offset, the flip from the pixels).

It also runs the detection train chain on 4 clips (draws and boxes) and the detection tutorial's
``ava_inference_transform`` on small uint8 clips followed by the reference's slow_r50_detection and
slowfast_r50_detection, with weights randomised as pytorchvideo_b200.testing does, and stores their logits.  Inputs
are regenerated from seeds; the file holds outputs, draws and checksums only.

    PYTHONPATH=<reference checkout> python oracle/gen_golden_boxes.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))

GOLD = os.path.join(ROOT, "tests", "golden", "boxes.pt")


def _np(b):
    return b.numpy() if torch.is_tensor(b) else np.asarray(b)


def stated_clip(b, h, w):
    t = b.dtype.type
    out = b.copy()
    out[:, [0, 2]] = np.minimum(t(w - 1.0), np.maximum(t(0.0), b[:, [0, 2]]))
    out[:, [1, 3]] = np.minimum(t(h - 1.0), np.maximum(t(0.0), b[:, [1, 3]]))
    return out


def stated_scale(b, h, w, new_h, new_w):
    t = b.dtype.type
    return b * t(float(new_h) / h if w < h else float(new_w) / w)


def stated_crop(b, y, x):
    t = b.dtype.type
    out = b.copy()
    out[:, [0, 2]] = b[:, [0, 2]] - t(x)
    out[:, [1, 3]] = b[:, [1, 3]] - t(y)
    return out


def stated_flip(b, w):
    t = b.dtype.type
    out = b.copy()
    out[:, 0] = (t(w) - b[:, 2]) - t(1)
    out[:, 2] = (t(w) - b[:, 0]) - t(1)
    return out


def run_functional(RF, TS):
    out = {}
    for name, (fn, (H, W), K, kw) in TS.BOX_FUNCTIONAL_CASES.items():
        for dtype in (torch.float32, torch.float64):
            seed, images, boxes = TS.box_case_inputs(name, dtype)
            b_in = boxes.numpy().copy()
            torch.manual_seed(seed)
            np.random.seed(seed)
            res = TS.call_box_case(RF, name, images, boxes.clone())
            draws = {}
            if fn in ("clip_boxes_to_image", "crop_boxes"):
                got = _np(res)
                want = stated_clip(b_in, H, W) if fn == "clip_boxes_to_image" else \
                    stated_crop(b_in, kw["y_offset"], kw["x_offset"])
            elif fn in ("short_side_scale_with_boxes", "random_short_side_scale_with_boxes"):
                img, got = res[0], _np(res[1])
                nh, nw = img.shape[2], img.shape[3]
                draws["new_hw"] = (nh, nw)
                want = stated_scale(b_in, H, W, nh, nw)
            elif fn in ("random_crop_with_boxes", "uniform_crop_with_boxes"):
                if torch.is_tensor(res):           # random_crop_with_boxes on a size x size clip: the clip alone
                    assert res is images
                    draws["offset"], got, want = None, None, None
                else:
                    img, got = res[0], _np(res[1])
                    y, x = divmod(img.storage_offset(), W)
                    draws["offset"] = (y, x)
                    want = stated_clip(stated_crop(b_in, y, x), img.shape[2], img.shape[3])
            else:
                img, got = res[0], _np(res[1])
                flip = not (img is images)
                if flip:
                    assert torch.equal(img, images.flip(-1))
                draws["flip"] = flip
                want = stated_flip(b_in, W) if flip else b_in
            if want is not None:
                assert got.dtype == want.dtype and np.array_equal(got, want, equal_nan=True), (name, dtype)
            out[(name, str(dtype))] = {"boxes": None if got is None else torch.from_numpy(np.ascontiguousarray(got)),
                                       "draws": draws}
        print("%-28s ok  %s" % (name, out[(name, "torch.float32")]["draws"]), flush=True)
    return out


def run_train_chain(RF, TS):
    c = TS.BOX_TRAIN_CHAIN
    clips, boxes = TS.train_chain_inputs()
    torch.manual_seed(c["seed"])
    np.random.seed(c["seed"])
    draws, outs, rois = [], [], []
    for b in range(clips.shape[0]):
        x = RF.uniform_temporal_subsample(clips[b], c["num_samples"]).float() / 255.0
        bx = RF.clip_boxes_to_image(boxes[b].clone(), x.shape[2], x.shape[3])
        x, bx = RF.random_short_side_scale_with_boxes(x, bx, *c["random_short_side"])
        side_hw = (x.shape[2], x.shape[3])
        W1 = x.shape[3]
        x, bx = RF.random_crop_with_boxes(x, c["crop"], bx)
        off = divmod(x.storage_offset(), W1)
        flipped, bx = RF.horizontal_flip_with_boxes(c["hflip_prob"], x, bx)
        flip = flipped is not x
        bx = RF.clip_boxes_to_image(bx, flipped.shape[2], flipped.shape[3])
        draws.append({"new_hw": side_hw, "offset": off, "flip": flip})
        outs.append(bx.clone())
        rois.append(torch.cat([torch.full((bx.shape[0], 1), float(b)), bx.float()], 1))
    print("train chain ok  %s" % draws, flush=True)
    return {"draws": draws, "boxes": outs, "rois": torch.cat(rois, 0)}


def ava_inference_transform(RF, clip, boxes, num_frames, crop_size, data_mean, data_std, slow_fast_alpha):
    """The detection tutorial's transform (website/docs/tutorial_torchhub_detection_inference.md), with torchvision's
    video ``normalize`` written out (clip.sub_(mean).div_(std) per channel)."""
    boxes = np.array(boxes)
    clip = RF.uniform_temporal_subsample(clip, num_frames)
    clip = clip.float()
    clip = clip / 255.0
    height, width = clip.shape[2], clip.shape[3]
    boxes = RF.clip_boxes_to_image(boxes, height, width)
    clip, boxes = RF.short_side_scale_with_boxes(clip, size=crop_size, boxes=boxes)
    mean = torch.as_tensor(np.array(data_mean, dtype=np.float32))
    std = torch.as_tensor(np.array(data_std, dtype=np.float32))
    clip = clip.clone().sub_(mean[:, None, None, None]).div_(std[:, None, None, None])
    boxes = RF.clip_boxes_to_image(boxes, clip.shape[2], clip.shape[3])
    if slow_fast_alpha is not None:
        fast_pathway = clip
        slow_pathway = torch.index_select(clip, 1, torch.linspace(0, clip.shape[1] - 1,
                                                                  clip.shape[1] // slow_fast_alpha).long())
        clip = [slow_pathway, fast_pathway]
    return clip, torch.from_numpy(boxes)


def run_tutorial(RF, TS):
    import pytorchvideo.models.hub as RH
    import pytorchvideo_b200.models.hub as PH
    c = TS.BOX_TUTORIAL
    out = {}
    for case, (hub, _, n_frames, alpha) in TS.BOX_TUTORIAL_CASES.items():
        clips, boxes = TS.tutorial_inputs(case)
        mine = TS.build_tutorial_model(case, PH)
        ref = getattr(RH, hub)(pretrained=False, head_activation=None)
        ref.load_state_dict(mine.state_dict(), strict=True)
        ref.eval()
        inputs, rois = [], []
        for b in range(clips.shape[0]):
            x, bx = ava_inference_transform(RF, clips[b], boxes[b].numpy(), n_frames, c["crop_size"], c["mean"],
                                            c["std"], alpha)
            inputs.append(x)
            rois.append(torch.cat([torch.full((bx.shape[0], 1), float(b)), bx], 1))
        rois = torch.cat(rois, 0)
        if alpha is None:
            net_in = torch.stack(inputs)
        else:
            net_in = [torch.stack([x[0] for x in inputs]), torch.stack([x[1] for x in inputs])]
        with torch.no_grad():
            logits = ref(list(net_in) if alpha else net_in, rois)
        out[case] = {"logits": logits.clone(), "rois": rois.clone(), "state_checksum": TS.state_checksum(mine),
                     "input_checksum": TS.tensor_checksum(torch.cat([t.reshape(-1) for t in (net_in if alpha else [net_in])]))}
        print("%-24s ok  logits %s  range [%.4f, %.4f]" % (case, tuple(logits.shape), float(logits.min()),
                                                        float(logits.max())), flush=True)
    return out


def main():
    import pytorchvideo.transforms.functional as RF
    from pytorchvideo_b200 import testing as TS
    out = {"functional": run_functional(RF, TS), "train_chain": run_train_chain(RF, TS),
           "tutorial": run_tutorial(RF, TS), "torch": torch.__version__, "numpy": np.__version__}
    torch.save(out, GOLD)
    print("wrote", GOLD)


if __name__ == "__main__":
    main()
