"""Golden vectors of MixUp, CutMix and MixVideo (tests/golden/mix.pt).

Runs the reference's own modules on the CPU under fixed seeds, on float32, float16 and uint8 batches of odd and even
size, with and without label smoothing, with one-hot labels and with audio.  For every case it asserts that
oracle/mix_ref.py makes the same draws and the same outputs bit for bit, and that this package's host sampler makes
the same draws (lambda, box, branch).  Writes the inputs, the draws and the reference outputs.  Runs only where the
reference package is importable: put its checkout on PYTHONPATH.

    PYTHONPATH=<reference checkout> python oracle/gen_golden_mix.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))

GOLD = os.path.join(ROOT, "tests", "golden", "mix.pt")
K = 10


def batch(shape, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    if dtype == torch.uint8:
        return torch.randint(0, 256, shape, generator=g, dtype=torch.uint8)
    return (torch.randn(shape, generator=g) * 1.5).to(dtype)     # normalised-clip range, signs mixed


def labels_for(B, seed, one_hot):
    g = torch.Generator().manual_seed(1000 + seed)
    if one_hot:
        return torch.softmax(torch.randn(B, K, generator=g) * 3, dim=1)   # float32 soft rows
    return torch.randint(0, K, (B,), generator=g)


def package_draws(mod, video_shape, audio_shape=None):
    """The draws of one call of this package's module ``mod`` (MixUp, CutMix or MixVideo) on torch's global RNG."""
    from pytorchvideo_b200.transforms import mix as M
    if isinstance(mod, M.MixUp):
        return {"lam": float(mod.sample())}
    if isinstance(mod, M.CutMix):
        lam, box, lam_c, abox = mod.sample(video_shape, audio_shape)
        return {"lam": float(lam), "box": box, "lam_c": lam_c, "audio_box": abox}
    if mod.use_cutmix():
        return dict(package_draws(mod.cutmix, video_shape), branch="cutmix")
    return dict(package_draws(mod.mixup, video_shape), branch="mixup")


def run_case(kind, kw, seed, video, labels, audio=None):
    from pytorchvideo.transforms import mix as R
    from oracle import mix_ref as O
    ref_mod = getattr(R, kind)(**kw)
    torch.manual_seed(seed)
    v, a = video.clone(), None if audio is None else audio.clone()
    res = ref_mod(v, labels.clone(), **({} if a is None else {"x_audio": a}))
    ref_v, ref_l = res[0], res[-1]
    ref_a = res[1] if a is not None else None
    assert ref_v is v and (a is None or ref_a is a)              # in place, the same tensors returned

    torch.manual_seed(seed)
    ls, nc, oh = kw.get("label_smoothing", 0.0), kw.get("num_classes", 400), kw.get("one_hot", False)
    if kind == "MixVideo":
        o_v, o_l, draws = O.mixvideo_call(video, labels, kw.get("cutmix_prob", 0.5), kw.get("mixup_alpha", 1.0),
                                          kw.get("cutmix_alpha", 1.0), ls, nc, oh)
        o_a = None
    else:
        call = O.mixup_call if kind == "MixUp" else O.cutmix_call
        o_v, o_a, o_l, draws = call(video, labels, kw.get("alpha", 1.0), ls, nc, oh, audio)
    assert o_v.dtype == ref_v.dtype and torch.equal(o_v, ref_v), (kind, kw, seed, "video")
    assert o_l.dtype == ref_l.dtype and torch.equal(o_l, ref_l), (kind, kw, seed, "labels", o_l.dtype, ref_l.dtype)
    if audio is not None:
        assert torch.equal(o_a, ref_a), (kind, kw, seed, "audio")

    from pytorchvideo_b200.transforms import mix as M
    mod = getattr(M, kind)(**kw)
    torch.manual_seed(seed)
    pk = package_draws(mod, video.shape, None if audio is None else audio.shape)
    assert pk == draws, (kind, kw, seed, pk, draws)
    return {"kind": kind, "kwargs": kw, "seed": seed, "video": video, "audio": audio, "labels": labels,
            "draws": draws, "out_video": ref_v.clone(), "out_audio": None if ref_a is None else ref_a.clone(),
            "out_labels": ref_l.clone()}


def find_seed(start, pred, kw, shape):
    """The first seed from ``start`` whose CutMix draws satisfy pred(box, H, W)."""
    from pytorchvideo_b200.transforms import mix as M
    for s in range(start, start + 10000):
        torch.manual_seed(s)
        _, box, _, _ = M.CutMix(alpha=kw.get("alpha", 1.0)).sample(shape)
        if pred(box, shape[-2], shape[-1]):
            return s
    raise RuntimeError("no seed found")


def main():
    cases = []
    shapes = {4: (4, 3, 2, 9, 11), 5: (5, 3, 2, 9, 11)}
    seed = 100
    for dt in (torch.float32, torch.float16):
        for B in (4, 5):
            for ls in (0.0, 0.1):
                seed += 1
                cases.append(run_case("MixUp", dict(alpha=0.8, label_smoothing=ls, num_classes=K), seed,
                                      batch(shapes[B], dt, seed), labels_for(B, seed, False)))
        seed += 1
        cases.append(run_case("MixUp", dict(alpha=0.8, num_classes=K, one_hot=True), seed, batch(shapes[5], dt, seed),
                              labels_for(5, seed, True)))
        seed += 1
        cases.append(run_case("MixUp", dict(label_smoothing=0.1, num_classes=K), seed, batch((4, 3, 9, 11), dt, seed),
                              labels_for(4, seed, False), audio=batch((4, 1, 6, 7), dt, seed + 1)))
    for dt in (torch.float32, torch.float16, torch.uint8):
        for B in (4, 5):
            for ls in (0.0, 0.1):
                seed += 1
                cases.append(run_case("CutMix", dict(label_smoothing=ls, num_classes=K), seed,
                                      batch(shapes[B], dt, seed), labels_for(B, seed, False)))
        seed += 1
        cases.append(run_case("CutMix", dict(num_classes=K, one_hot=True), seed, batch(shapes[4], dt, seed),
                              labels_for(4, seed, True)))
        seed += 1
        cases.append(run_case("CutMix", dict(label_smoothing=0.1, num_classes=K), seed, batch((5, 3, 9, 11), dt, seed),
                              labels_for(5, seed, False), audio=batch((5, 1, 6, 7), dt, seed + 1)))
    # edge boxes: empty (lam near 1), clipped at the top-left and at the bottom-right edge
    kw = dict(alpha=0.1, label_smoothing=0.1, num_classes=K)
    for name, pred in [("empty", lambda b, h, w: b[0] == b[1] or b[2] == b[3]),
                       ("clip_lo", lambda b, h, w: b[0] == 0 and b[2] == 0 and 0 < b[1] < h and 0 < b[3] < w),
                       ("clip_hi", lambda b, h, w: b[1] == h and b[3] == w and 0 < b[0] and 0 < b[2])]:
        s = find_seed(500, pred, kw, shapes[5])
        c = run_case("CutMix", kw, s, batch(shapes[5], torch.float32, s), labels_for(5, s, False))
        c["edge"] = name
        cases.append(c)
    # MixVideo: the MViT recipe's arguments; seeds reach both branches
    for s in range(700, 706):
        kw = dict(cutmix_prob=0.5, mixup_alpha=0.8, cutmix_alpha=1.0, label_smoothing=0.1, num_classes=K)
        cases.append(run_case("MixVideo", kw, s, batch(shapes[5], torch.float32, s), labels_for(5, s, False)))
    for s in range(710, 713):
        kw = dict(cutmix_prob=0.0, label_smoothing=0.0, num_classes=K, one_hot=True)
        cases.append(run_case("MixVideo", kw, s, batch(shapes[4], torch.float16, s), labels_for(4, s, True)))
    branches = {c["draws"]["branch"] for c in cases if c["kind"] == "MixVideo"}
    assert branches == {"mixup", "cutmix"}, branches
    torch.save({"cases": cases}, GOLD)
    print("wrote", GOLD, os.path.getsize(GOLD), "bytes;", len(cases), "cases")


if __name__ == "__main__":
    main()
