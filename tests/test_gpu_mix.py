"""MixUp, CutMix and MixVideo: host draws, argument checks and the oracle on the CPU, the in-place kernels on the GPU.

Goldens (tests/golden/mix.pt, oracle/gen_golden_mix.py) hold the reference's outputs and draws under fixed seeds.
Every GPU result is held to bit equality: MixUp rounds each eager op of the reference once, CutMix is a copy, and the
labels are the reference's float32 products and sum.
"""
import ctypes
import os
import re
import subprocess
import tempfile

import pytest
import torch

from oracle import mix_ref as O
from pytorchvideo_b200 import _lib as L
from pytorchvideo_b200 import testing as TS
from pytorchvideo_b200.transforms import CutMix, FusedClipTransform, MixUp, MixVideo, Permute
from pytorchvideo_b200.transforms import functional as Fv
from pytorchvideo_b200.transforms import mix as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pytorchvideo_b200", "csrc")
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "mix.pt"), weights_only=False)["cases"]


def _dev():
    return torch.device("cuda:0")


def _case_id(c):
    return "%s-%d-%s-B%d" % (c["kind"], c["seed"], str(c["video"].dtype).split(".")[-1], c["video"].shape[0])


def _module(c):
    return getattr(M, c["kind"])(**c["kwargs"])


def _draws(mod, video_shape, audio_shape=None):
    """The draws of one call of ``mod`` on torch's global RNG, in the goldens' format."""
    if isinstance(mod, MixUp):
        return {"lam": float(mod.sample())}
    if isinstance(mod, CutMix):
        lam, box, lam_c, abox = mod.sample(video_shape, audio_shape)
        return {"lam": float(lam), "box": box, "lam_c": lam_c, "audio_box": abox}
    if mod.use_cutmix():
        return dict(_draws(mod.cutmix, video_shape), branch="cutmix")
    return dict(_draws(mod.mixup, video_shape), branch="mixup")


# ---- CPU: oracle, host draws, goldens' coverage ---------------------------------------------------------------------
def _oracle_call(c, video, labels, audio=None):
    kw = c["kwargs"]
    ls, nc, oh = kw.get("label_smoothing", 0.0), kw.get("num_classes", 400), kw.get("one_hot", False)
    torch.manual_seed(c["seed"])
    if c["kind"] == "MixVideo":
        v, lab, d = O.mixvideo_call(video, labels, kw.get("cutmix_prob", 0.5), kw.get("mixup_alpha", 1.0),
                                    kw.get("cutmix_alpha", 1.0), ls, nc, oh)
        return v, None, lab, d
    call = O.mixup_call if c["kind"] == "MixUp" else O.cutmix_call
    return call(video, labels, kw.get("alpha", 1.0), ls, nc, oh, audio)


@pytest.mark.parametrize("case", GOLD, ids=[_case_id(c) for c in GOLD])
def test_oracle_reproduces_golden(case):
    v, a, lab, draws = _oracle_call(case, case["video"], case["labels"], case["audio"])
    assert v.dtype == case["out_video"].dtype and torch.equal(v, case["out_video"])
    assert lab.dtype == case["out_labels"].dtype and torch.equal(lab, case["out_labels"])
    if case["audio"] is not None:
        assert torch.equal(a, case["out_audio"])
    assert draws == case["draws"]


def test_host_draws_equal_recorded_draws():
    for c in GOLD:
        torch.manual_seed(c["seed"])
        got = _draws(_module(c), c["video"].shape, None if c["audio"] is None else c["audio"].shape)
        assert got == c["draws"], (_case_id(c), got, c["draws"])


def test_goldens_cover_the_edges():
    kinds = {(c["kind"], c["video"].dtype, c["video"].shape[0] % 2) for c in GOLD}
    for dt in (torch.float32, torch.float16):
        assert ("MixUp", dt, 0) in kinds and ("MixUp", dt, 1) in kinds
    for dt in (torch.float32, torch.float16, torch.uint8):
        assert ("CutMix", dt, 0) in kinds and ("CutMix", dt, 1) in kinds
    assert {c["draws"]["branch"] for c in GOLD if c["kind"] == "MixVideo"} == {"mixup", "cutmix"}
    boxes = [c["draws"]["box"] for c in GOLD if "box" in c["draws"]]
    assert any(b[0] == b[1] or b[2] == b[3] for b in boxes)                       # an empty box
    assert {c.get("edge") for c in GOLD} >= {"empty", "clip_lo", "clip_hi"}
    assert any(c["audio"] is not None for c in GOLD if c["kind"] == "MixUp")
    assert any(c["audio"] is not None for c in GOLD if c["kind"] == "CutMix")
    assert any(c["kwargs"].get("one_hot") for c in GOLD)
    assert {c["kwargs"].get("label_smoothing", 0.0) for c in GOLD} == {0.0, 0.1}


def test_one_hot_values_are_convert_to_one_hots():
    lab = torch.tensor([2, 0, 6])
    rows = O.one_hot_rows(lab, 7, 0.1)
    off = torch.tensor(0.1 / 7, dtype=torch.float32)
    assert rows.dtype == torch.float32 and torch.equal(rows[0, 2], torch.tensor(1.0 - 0.1 + 0.1 / 7, dtype=torch.float32))
    assert torch.equal(rows[1, 1], off)


# ---- CPU: argument checks -------------------------------------------------------------------------------------------
def test_errors_without_a_device():
    x = torch.zeros(4, 3, 2, 8, 8)
    lab = torch.zeros(4, dtype=torch.int64)
    with pytest.raises(AssertionError):
        MixUp()(torch.zeros(1, 3, 2, 8, 8), lab[:1])                     # B = 1
    with pytest.raises(AssertionError):
        CutMix()(torch.zeros(1, 3, 2, 8, 8), lab[:1])
    with pytest.raises(AssertionError):
        CutMix()(torch.zeros(4, 3, 8), lab)                               # CutMix rank
    with pytest.raises(AssertionError):
        CutMix()(torch.zeros(4, 3, 2, 2, 8, 8), lab)
    with pytest.raises(AssertionError):
        MixVideo(cutmix_prob=1.5)
    with pytest.raises(AssertionError):
        MixVideo(cutmix_prob=-0.1)
    with pytest.raises(RuntimeError):
        MixUp()(x.to(torch.uint8), lab)                                    # MixUp on uint8
    with pytest.raises(RuntimeError):
        CutMix()(x.double(), lab)
    with pytest.raises(RuntimeError):
        MixUp()(torch.zeros(1, 3, 2, 8, 8).expand(4, -1, -1, -1, -1), lab)  # self-overlapping batch
    with pytest.raises(RuntimeError):
        CutMix()(torch.zeros(4, 3, 2, 8, 1).expand(-1, -1, -1, -1, 8), lab)
    with pytest.raises(TypeError):
        MixVideo()(x, lab, x_audio=x.clone())
    with pytest.raises(RuntimeError):                                     # CutMix branch is built without one_hot
        MixVideo(cutmix_prob=1.0, num_classes=10, one_hot=True)(x, torch.full((4, 10), 0.1))
    with pytest.raises(RuntimeError):
        MixUp()(x, lab)                                                    # CPU tensors
    with pytest.raises(RuntimeError):
        CutMix()(x, lab)
    with pytest.raises(RuntimeError):
        Fv.convert_to_one_hot(lab, 10)
    with pytest.raises(RuntimeError):
        MixUp()(x, lab.int())                                              # label dtype
    with pytest.raises(RuntimeError):
        MixUp(one_hot=True)(x, torch.zeros(4, 10, dtype=torch.float64))


def test_overlap_check():
    x = torch.zeros(4, 3, 2, 8, 8)
    assert not M._overlaps(x)
    assert not M._overlaps(x.contiguous(memory_format=torch.channels_last_3d))
    assert not M._overlaps(x.permute(0, 2, 1, 3, 4))
    assert not M._overlaps(x[:, :, :, ::2, 1:])
    assert M._overlaps(x[:1].expand(4, -1, -1, -1, -1))
    assert M._overlaps(torch.zeros(10).as_strided((4, 4), (2, 1)))


def test_descriptor_pads_to_four_dims():
    x = torch.zeros(4, 3, 8, 8, dtype=torch.float16).permute(0, 1, 3, 2)
    d = M._mix_desc(x)
    assert (d.B, d.dtype, list(d.size), list(d.stride), d.s_batch) == (4, L.PV_F16, [1, 3, 8, 8], [0, 64, 1, 8], 192)


def test_struct_sizes_match_header():
    probe = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "pv_b200.h"
    int main(){ printf("%zu %zu %zu %zu\n", sizeof(pv_mix_desc), sizeof(pv_mix_label_desc),
                       offsetof(pv_mix_desc, s_batch), offsetof(pv_mix_label_desc, s_row)); return 0; }'''
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "p.c")
        open(c, "w").write(probe)
        exe = os.path.join(td, "p")
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe], check=True)
        got = [int(v) for v in subprocess.run([exe], capture_output=True, text=True).stdout.split()]
    assert got == [ctypes.sizeof(L.MixDesc), ctypes.sizeof(L.MixLabelDesc), L.MixDesc.s_batch.offset,
                   L.MixLabelDesc.s_row.offset]


# ---- CPU: instance ledger -------------------------------------------------------------------------------------------
MIX_INSTANCES = {"mixup_kernel<float>", "mixup_kernel<__half>", "mixup_vec_kernel<float>", "mixup_vec_kernel<__half>",
                 "cutmix_kernel<1>", "cutmix_kernel<2>", "cutmix_kernel<4>", "mix_labels_kernel<index>",
                 "mix_labels_kernel<onehot>"}
# which GPU test reaches each instance
LEDGER = {
    "mixup_kernel<float>": "test_gpu_golden[MixUp-101-float32-B4]",
    "mixup_kernel<__half>": "test_gpu_golden[MixUp-107-float16-B4]",
    "mixup_vec_kernel<float>": "test_gpu_strided_inputs[float32]",
    "mixup_vec_kernel<__half>": "test_gpu_strided_inputs[float16]",
    "cutmix_kernel<1>": "test_gpu_golden[CutMix-126-uint8-B4]",
    "cutmix_kernel<2>": "test_gpu_golden[CutMix-119-float16-B4]",
    "cutmix_kernel<4>": "test_gpu_golden[CutMix-113-float32-B4]",
    "mix_labels_kernel<index>": "test_gpu_golden[MixUp-101-float32-B4]",
    "mix_labels_kernel<onehot>": "test_gpu_golden[MixUp-105-float32-B5]",
}


def test_instance_ledger():
    src = open(os.path.join(CSRC, "pv_mix.cu")).read()
    assert set(re.findall(r'PV_LAUNCH_OK\("([^"]+)"\)', src)) == MIX_INSTANCES
    assert set(LEDGER) == MIX_INSTANCES
    ids = {"test_gpu_golden[%s]" % _case_id(c) for c in GOLD}
    for inst, test in LEDGER.items():
        assert test in ids or not test.startswith("test_gpu_golden"), (inst, test)
        if test.startswith("test_gpu_golden"):
            c = next(c for c in GOLD if "test_gpu_golden[%s]" % _case_id(c) == test)
            assert inst in _expected_launches(c, c["video"], c["audio"]), (inst, test)


# ---- GPU ------------------------------------------------------------------------------------------------------------
_TAG = {torch.float32: "float", torch.float16: "__half"}
_ES = {torch.float32: 4, torch.float16: 2, torch.uint8: 1}


def _mixup_instance(x):
    """The MixUp kernel pv_mixup picks: 16-byte vectors when each clip is one dense, 16-byte-aligned block."""
    es = _ES[x.dtype]
    d = M._mix_desc(x)
    dims = sorted((s, n) for n, s in zip(d.size, d.stride) if n > 1)
    expect, dense = 1, True
    for s, n in dims:
        dense = dense and s == expect
        expect *= n
    vec = dense and (expect * es) % 16 == 0 and (d.s_batch * es) % 16 == 0 and x.data_ptr() % 16 == 0
    return ("mixup_vec_kernel<%s>" if vec else "mixup_kernel<%s>") % _TAG[x.dtype]


def _expected_launches(c, video, audio):
    onehot = c["kwargs"].get("one_hot", False) and c["draws"].get("branch") != "cutmix"
    want = {"mix_labels_kernel<onehot>" if onehot else "mix_labels_kernel<index>": 1}
    cut = c["kind"] == "CutMix" or c["draws"].get("branch") == "cutmix"
    for x, box in ((video, c["draws"].get("box")), (audio, c["draws"].get("audio_box"))):
        if x is None:
            continue
        if cut:
            if box[0] != box[1] and box[2] != box[3]:
                name = "cutmix_kernel<%d>" % _ES[x.dtype]
                want[name] = want.get(name, 0) + 1
        else:
            name = _mixup_instance(x)
            want[name] = want.get(name, 0) + 1
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("case", GOLD, ids=[_case_id(c) for c in GOLD])
def test_gpu_golden(case):
    dev = _dev()
    v = case["video"].to(dev)
    a = None if case["audio"] is None else case["audio"].to(dev)
    lab = case["labels"].to(dev)
    ptr = v.data_ptr()
    mod = _module(case)
    torch.manual_seed(case["seed"])
    out, launched = TS.launched_kernels(lambda: mod(v, lab, **({} if a is None else {"x_audio": a})))
    assert len(out) == (2 if a is None else 3)
    assert out[0] is v and v.data_ptr() == ptr
    if a is not None:
        assert out[1] is a
        assert torch.equal(a.cpu(), case["out_audio"])
    assert launched == _expected_launches(case, v, a), launched
    assert v.dtype == case["out_video"].dtype and torch.equal(v.cpu(), case["out_video"])
    got = out[-1]
    assert got.dtype == case["out_labels"].dtype and got.device == dev and torch.equal(got.cpu(), case["out_labels"])


def _clips(B, dtype, T=4, H=16, W=24, seed=0):
    g = torch.Generator().manual_seed(seed)
    if dtype == torch.uint8:
        return torch.randint(0, 256, (B, 3, T, H, W), generator=g, dtype=torch.uint8)
    return (torch.randn(B, 3, T, H, W, generator=g) * 1.5).to(dtype)


def _layouts(x):
    """The same (B, C, T, H, W) values as contiguous, channels-last and a Permute view of (B, T, C, H, W) storage."""
    dev = _dev()
    btchw = x.permute(0, 2, 1, 3, 4).contiguous().to(dev)
    return {"contiguous": x.to(dev),
            "channels_last": x.to(dev).contiguous(memory_format=torch.channels_last_3d),
            "permute": Permute((0, 2, 1, 3, 4))(btchw)}


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.uint8], ids=["float32", "float16", "uint8"])
def test_gpu_strided_inputs(dtype):
    x = _clips(5, dtype)
    lab = torch.tensor([3, 1, 4, 1, 5])
    mods = [("cutmix", lambda: CutMix(num_classes=7, label_smoothing=0.1))]
    if dtype != torch.uint8:
        mods.append(("mixup", lambda: MixUp(alpha=0.8, num_classes=7)))
    for name, make in mods:
        torch.manual_seed(21)
        want_v, _, want_l, _ = (O.cutmix_call if name == "cutmix" else O.mixup_call)(
            x, lab, 1.0 if name == "cutmix" else 0.8, 0.1 if name == "cutmix" else 0.0, 7)
        for layout, inp in _layouts(x).items():
            torch.manual_seed(21)
            out, launched = TS.launched_kernels(lambda: make()(inp, lab.to(_dev())))
            assert out[0] is inp
            if name == "mixup":                                        # each layout is one dense block per clip
                assert launched == {"mixup_vec_kernel<%s>" % _TAG[dtype]: 1, "mix_labels_kernel<index>": 1}, launched
            assert torch.equal(inp.cpu(), want_v), (name, layout)
            assert torch.equal(out[1].cpu(), want_l), (name, layout)
    # a slice is not one dense block: the general strided path
    if dtype != torch.uint8:
        base = _clips(5, dtype, W=31).to(_dev())
        view = base[..., 2:29:2]
        torch.manual_seed(4)
        want_v = O.mixup_call(view.cpu(), lab, 0.8, 0.0, 7)[0]
        torch.manual_seed(4)
        out, launched = TS.launched_kernels(lambda: MixUp(alpha=0.8, num_classes=7)(view, lab.to(_dev())))
        assert launched.get("mixup_kernel<%s>" % _TAG[dtype]) == 1, launched
        assert torch.equal(view.cpu(), want_v)
        rest = base.clone()
        rest[..., 2:29:2] = 0
        untouched = _clips(5, dtype, W=31)
        untouched[..., 2:29:2] = 0
        assert torch.equal(rest.cpu(), untouched)                  # elements outside the view are not written


@pytest.mark.gpu
def test_gpu_memory_does_not_grow_with_the_batch():
    dev = _dev()
    B, K = 16, 400
    lab = torch.randint(0, K, (B,)).to(dev)
    for dtype, make in ((torch.float32, lambda: MixUp()), (torch.float16, lambda: MixUp()),
                        (torch.uint8, lambda: CutMix())):
        x = _clips(B, dtype, T=8, H=64, W=64).to(dev)
        make()(x, lab)                                              # warm the allocator's small pool
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated(dev)
        torch.manual_seed(0)
        out = make()(x, lab)
        torch.cuda.synchronize()
        grew = torch.cuda.memory_allocated(dev) - before
        assert grew <= B * K * 4 + 1024, (dtype, grew)             # the labels plus the allocator's rounding
        del out


@pytest.mark.gpu
def test_gpu_bad_labels_leave_the_batch_unchanged():
    dev = _dev()
    x = _clips(4, torch.float32).to(dev)
    keep = x.clone()
    for mod in (MixUp(num_classes=10), CutMix(num_classes=10), MixVideo(num_classes=10)):
        with pytest.raises(AssertionError):
            mod(x, torch.tensor([1, 10, 2, 3], device=dev))
        with pytest.raises(RuntimeError):
            mod(x, torch.tensor([1, -1, 2, 3], device=dev))
        assert torch.equal(x, keep)
    with pytest.raises(AssertionError):
        MixUp(num_classes=10, label_smoothing=1.0)(x, torch.tensor([1, 2, 2, 3], device=dev))
    with pytest.raises(RuntimeError):
        MixUp()(x, torch.tensor([1, 2, 2, 3]))                     # labels on another device
    assert torch.equal(x, keep)


@pytest.mark.gpu
def test_gpu_convert_to_one_hot():
    dev = _dev()
    lab = torch.tensor([3, 0, 9, 3, 5])
    got, launched = TS.launched_kernels(lambda: Fv.convert_to_one_hot(lab.to(dev), 10))
    assert launched == {"mix_labels_kernel<index>": 1}
    want = torch.zeros(5, 10, dtype=torch.int64)
    want[torch.arange(5), lab] = 1
    assert got.dtype == torch.int64 and torch.equal(got.cpu(), want)
    got = Fv.convert_to_one_hot(lab.to(dev), 10, 0.2)
    assert got.dtype == torch.float32 and torch.equal(got.cpu(), O.one_hot_rows(lab, 10, 0.2))
    with pytest.raises(AssertionError):
        Fv.convert_to_one_hot(lab.to(dev), 9)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["float32", "float16"])
def test_gpu_repeat_is_deterministic(dtype):
    x = _clips(6, dtype, T=8, H=32, W=32)
    lab = torch.tensor([0, 1, 2, 3, 4, 5])
    outs = []
    for _ in range(2):
        for seed in (1, 2, 3, 4):
            v = x.to(_dev())
            torch.manual_seed(seed)
            _, lo = MixVideo(mixup_alpha=0.8, label_smoothing=0.1, num_classes=6)(v, lab.to(_dev()))
            outs.append((v.cpu(), lo.cpu()))
    for (a, la), (b, lb) in zip(outs[:4], outs[4:]):
        assert torch.equal(a, b) and torch.equal(la, lb)


@pytest.mark.gpu
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.float16], ids=["float32", "float16"])
def test_gpu_fused_transform_then_mixvideo(out_dtype):
    """The MViT recipe's batch step after its per-clip step: FusedClipTransform (random resized crop) makes the batch,
    MixVideo mixes it in place; the oracle (pinned to the reference by the goldens) runs on a CPU copy."""
    dev = _dev()
    B = 5
    u8 = torch.stack([TS.synthetic_u8_clip(12, 40, 52, seed=s) for s in range(B)]).to(dev)    # (B, 3, T, H, W)
    rrc = dict(target_height=24, target_width=32, scale=(0.08, 1.0), aspect_ratio=(0.75, 1.3333))
    tr = FusedClipTransform(8, (0.45,) * 3, (0.225,) * 3, random_resized_crop=rrc, hflip_prob=0.5, out_dtype=out_dtype)
    kw = dict(cutmix_prob=0.5, mixup_alpha=0.8, cutmix_alpha=1.0, label_smoothing=0.1, num_classes=10)
    lab = torch.tensor([7, 2, 9, 0, 2])
    branches = set()
    for seed in range(8):
        torch.manual_seed(seed)
        x = tr(u8)
        assert x.shape == (B, 3, 8, 24, 32) and x.dtype == out_dtype
        cpu = x.cpu()
        state = torch.get_rng_state()
        out, lo = MixVideo(**kw)(x, lab.to(dev))
        torch.set_rng_state(state)
        want, want_l, draws = O.mixvideo_call(cpu, lab, kw["cutmix_prob"], kw["mixup_alpha"], kw["cutmix_alpha"],
                                              kw["label_smoothing"], kw["num_classes"])
        branches.add(draws["branch"])
        assert out is x and torch.equal(x.cpu(), want) and torch.equal(lo.cpu(), want_l), (seed, draws)
    assert branches == {"mixup", "cutmix"}
