"""RandAugment and AugMix for video on the GPU (reference transforms/augmentations.py, rand_augment.py, augmix.py).

The host draws every random number from torch's global RNG with the reference's calls in the reference's order, so
under one seed the same ops and parameters are picked.  What reaches the GPU is one ``pv_aug_op`` per clip and layer
step: one ``pv_augment_apply`` launch per step for the whole batch, preceded by one ``pv_augment_stats`` launch when
some clip's op needs whole-frame statistics (AutoContrast, Equalize, AdjustContrast).
"""
import ctypes as C
import math

import numpy as np
import torch

from .. import _lib as L

MAX_LEVEL = 10
OP_NAMES = ("AdjustBrightness", "AdjustContrast", "AdjustSaturation", "AdjustSharpness", "AutoContrast", "Equalize",
            "Invert", "Rotate", "Posterize", "Solarize", "ShearX", "ShearY", "TranslateX", "TranslateY")
AUGMIX_OP_NAMES = ("AutoContrast", "Equalize", "Rotate", "Posterize", "Solarize", "ShearX", "ShearY", "TranslateX",
                   "TranslateY", "AdjustSaturation", "AdjustContrast", "AdjustBrightness", "AdjustSharpness")
_KIND = {"AdjustBrightness": 1, "AdjustContrast": 2, "AdjustSaturation": 3, "AdjustSharpness": 4, "AutoContrast": 5,
         "Equalize": 6, "Invert": 7, "Posterize": 8, "Solarize": 9, "Rotate": 10, "ShearX": 10, "ShearY": 10,
         "TranslateX": 10, "TranslateY": 10}
_NEEDS_STATS = {2, 5, 6}

# (base, range) of each op's argument at level 0 .. MAX_LEVEL
RANDAUG_MAX_PARAMS = {"AdjustBrightness": (1, 0.9), "AdjustContrast": (1, 0.9), "AdjustSaturation": (1, 0.9),
                      "AdjustSharpness": (1, 0.9), "AutoContrast": None, "Equalize": None, "Invert": None,
                      "Rotate": (0, 30), "Posterize": (4, 4), "Solarize": (1, 1), "ShearX": (0, 0.3),
                      "ShearY": (0, 0.3), "TranslateX": (0, 0.45), "TranslateY": (0, 0.45)}
AUGMIX_MAX_PARAMS = {"AutoContrast": None, "Equalize": None, "Rotate": (0, 30), "Posterize": (4, 4),
                     "Solarize": (1, 1), "ShearX": (0, 0.3), "ShearY": (0, 0.3), "TranslateX": (0, 1.0 / 3.0),
                     "TranslateY": (0, 1.0 / 3.0), "AdjustSaturation": (0.1, 1.8), "AdjustContrast": (0.1, 1.8),
                     "AdjustBrightness": (0.1, 1.8), "AdjustSharpness": (0.1, 1.8)}
DEFAULT_TRANSFORM_HPARAS = {"fill": (0.5, 0.5, 0.5)}
RANDAUG_SAMPLING_HPARAS = {"sampling_data_type": "int", "sampling_min": 0, "sampling_std": 0.5}
AUGMIX_SAMPLING_HPARAS = {"sampling_data_type": "float", "sampling_min": 0.1}


# ---- level -> argument (the reference's level functions) ---------------------------------------------------------
def _negate_half(v):
    return v if torch.rand(1).item() > 0.5 else -v


def _level_arg(kind, level, params):
    """kind: "neg" (increase, randomly negated), "inc", "dec_int", "dec"."""
    mag = (level / MAX_LEVEL) * params[1]
    if kind == "neg":
        return params[0] + _negate_half(mag)
    if kind == "inc":
        return params[0] + mag
    if kind == "dec_int":
        return params[0] - int(mag)
    return params[0] - mag


_RANDAUG_LEVEL = {"AdjustBrightness": "neg", "AdjustContrast": "neg", "AdjustSaturation": "neg",
                  "AdjustSharpness": "neg", "Rotate": "neg", "Posterize": "dec_int", "Solarize": "dec",
                  "ShearX": "neg", "ShearY": "neg", "TranslateX": "neg", "TranslateY": "neg"}
_AUGMIX_LEVEL = dict(_RANDAUG_LEVEL, AdjustSaturation="inc", AdjustContrast="inc", AdjustBrightness="inc",
                     AdjustSharpness="inc")


class _OpDraw:
    """One AugmentTransform of the reference: its probability check, magnitude sampling and level function."""

    def __init__(self, name, magnitude, prob, max_params, level_kinds, sampling_type, sampling_hparas):
        self.name, self.magnitude, self.prob = name, magnitude, prob
        self.params, self.level = max_params[name], level_kinds.get(name)
        self.sampling_type, self.hp = sampling_type, sampling_hparas

    def _magnitude(self):
        if self.sampling_type == "gaussian":
            return max(0, min(MAX_LEVEL, torch.normal(self.magnitude, self.hp["sampling_std"], size=(1,)).item()))
        if self.hp["sampling_data_type"] == "int":
            return torch.randint(self.hp["sampling_min"], self.magnitude + 1, size=(1,)).item()
        if self.hp["sampling_data_type"] == "float":
            return torch.rand(size=(1,)).item() * (self.magnitude - self.hp["sampling_min"]) + self.hp["sampling_min"]
        raise ValueError("sampling_data_type must be either 'int' or 'float'")

    def draw(self):
        """(name, argument or None), or None when the probability check skips the op."""
        if torch.rand(1).item() > self.prob:
            return None
        level = self._magnitude()
        return self.name, (_level_arg(self.level, level, self.params) if self.level is not None else None)


def _make_draws(names, magnitude, prob, max_params, level_kinds, transform_hparas, sampling_type, sampling_hparas):
    assert sampling_type in ("gaussian", "uniform")
    hp = transform_hparas or DEFAULT_TRANSFORM_HPARAS
    assert "fill" in hp
    if sampling_type == "gaussian":
        assert "sampling_std" in sampling_hparas
    else:
        assert "sampling_data_type" in sampling_hparas and "sampling_min" in sampling_hparas
        if sampling_hparas["sampling_data_type"] == "int":
            assert isinstance(sampling_hparas["sampling_min"], int)
        elif sampling_hparas["sampling_data_type"] == "float":
            assert isinstance(sampling_hparas["sampling_min"], (int, float))
    return [_OpDraw(n, magnitude, prob, max_params, level_kinds, sampling_type, sampling_hparas) for n in names], hp


def _sample_ops(draws, num_sample_op, randomly_sample_depth=False, replacement=False):
    """OpSampler.forward: randint for the depth (optional), multinomial over uniform weights, then each op's draws."""
    depth = torch.randint(1, num_sample_op + 1, (1,)).item() if randomly_sample_depth else num_sample_op
    index_list = torch.multinomial(torch.FloatTensor([1] * len(draws)), depth, replacement=replacement)
    return [draws[int(i)].draw() for i in index_list]


# ---- op -> pv_aug_op ----------------------------------------------------------------------------------------------
def rotate_matrix(angle):
    """torchvision rotate's inverse affine matrix about the centre (angle in degrees, counter-clockwise): the
    rotation by -angle, with no shear, scale or translation."""
    rot = math.radians(-angle)
    return [math.cos(rot), math.sin(rot), 0.0, -math.sin(rot), math.cos(rot), 0.0]


def affine_matrix(name, arg, h, w):
    """The 2x3 matrix the reference hands to the grid generator for a warp op on an h x w frame."""
    if name == "Rotate":
        return rotate_matrix(arg)
    if name == "ShearX":
        return [1, arg, h * arg / 2, 0, 1, 0]
    if name == "ShearY":
        return [1, 0, 0, arg, 1, w * arg / 2]
    if name == "TranslateX":
        return [1, 0, arg * w, 0, 1, 0]
    if name == "TranslateY":
        return [1, 0, 0, 0, 1, arg * h]
    raise ValueError(name)


def encode_op(op, dtype, h, w, fill):
    """pv_aug_op field values (kind, ival, ratio, omr, theta[6], fill[3]) of one drawn op, or the identity."""
    rec = [0, 0, 0.0, 0.0] + [0.0] * 6 + [float(f) for f in fill]
    if op is None:
        return rec
    name, arg = op
    kind = _KIND[name]
    u8 = dtype == torch.uint8
    if name in ("AdjustBrightness", "AdjustContrast", "AdjustSaturation", "AdjustSharpness"):
        if name == "AdjustSharpness" and (h <= 2 or w <= 2):
            return rec                                   # torchvision returns such frames unchanged
        ratio = float(arg)
        rec[0], rec[2], rec[3] = kind, ratio, 1.0 - ratio
    elif name == "Posterize":
        if arg >= 8:
            return rec
        if arg < 0:
            raise ValueError("Posterize bits must be in 0..8 (got %r)" % (arg,))
        rec[0], rec[1] = kind, (-int(2 ** (8 - arg))) & 0xFF
    elif name == "Solarize":
        if u8:
            thr = int(arg * 255.0)
            if thr > 255:
                raise TypeError("Threshold should be less than bound of img.")
            rec[0], rec[1] = kind, thr
        else:
            if arg > 1.0:
                raise TypeError("Threshold should be less than bound of img.")
            rec[0], rec[2] = kind, float(arg)
    elif kind == 10:
        theta = np.asarray(affine_matrix(name, arg, h, w), np.float32).reshape(2, 3)
        theta = theta / np.asarray([[0.5 * w], [0.5 * h]], np.float32)     # fp32, like the grid generator
        rec[0] = kind
        rec[4:10] = [float(v) for v in theta.reshape(-1)]
    else:
        rec[0] = kind
    return rec


def _ops_array(records):
    arr = (L.AugOp * len(records))()
    for a, r in zip(arr, records):
        a.kind, a.ival, a.ratio, a.omr = int(r[0]), int(r[1]), r[2], r[3]
        for i in range(6):
            a.theta[i] = r[4 + i]
        for i in range(3):
            a.fill[i] = r[10 + i]
    return arr


# ---- GPU execution --------------------------------------------------------------------------------------------------
def _check_clips(x):
    """(B, T, 3, H, W) view of a (T, 3, H, W) clip or a batch of them, and whether a batch dim was added."""
    if not torch.is_tensor(x) or x.dim() not in (4, 5):
        raise RuntimeError("expected a (T, C, H, W) clip or a (B, T, C, H, W) batch")
    if x.device.type != "cuda":
        raise RuntimeError("pytorchvideo_b200 transforms run on the GPU only (no CPU path)")
    if x.dtype not in (torch.uint8, torch.float32):
        raise RuntimeError("augmentation takes uint8 or float32 clips (got %s)" % x.dtype)
    squeeze = x.dim() == 4
    xb = x.unsqueeze(0) if squeeze else x
    if xb.shape[2] != 3:
        raise RuntimeError("augmentation needs 3-channel frames (got %d)" % xb.shape[2])
    return xb, squeeze


def _desc(x, n_clips, src_div):
    d = L.AugmentDesc()
    d.n_clips, d.src_div = n_clips, src_div
    d.T, d.C, d.H, d.W = x.shape[1], x.shape[2], x.shape[3], x.shape[4]
    d.s_clip, d.st, d.sc, d.sh, d.sw = (x.stride(i) for i in range(5))
    d.dtype = L.PV_U8 if x.dtype == torch.uint8 else L.PV_F32
    return d


def run_layers(x, plans, src_div=1, fill=(0.5, 0.5, 0.5)):
    """Apply plans[clip] = [op, op, ...] (drawn ops or None) to the (B, T, 3, H, W) clips ``x``; virtual clip k reads
    source clip k // src_div.  Returns a new contiguous (len(plans), T, 3, H, W) tensor of x's dtype."""
    lib = L.load()
    n, T, _, H, W = len(plans), x.shape[1], x.shape[2], x.shape[3], x.shape[4]
    dev = x.device
    steps = max((len(p) for p in plans), default=0)
    records = []
    for s in range(steps):
        records += [encode_op(p[s] if s < len(p) else None, x.dtype, H, W, fill) for p in plans]
    stream = torch.cuda.current_stream(dev).cuda_stream
    bufs = [torch.empty((n, T, 3, H, W), dtype=x.dtype, device=dev) for _ in range(min(steps, 2))]
    if steps == 0:
        out = torch.empty((n, T, 3, H, W), dtype=x.dtype, device=dev)
        records = [encode_op(None, x.dtype, H, W, fill)] * n
        steps, bufs = 1, [out]
    ops_host = _ops_array(records)
    ops_d = torch.frombuffer(bytearray(bytes(ops_host)), dtype=torch.uint8).to(dev)
    op_bytes = C.sizeof(L.AugOp) * n
    stats = None
    src, div, cur = x, src_div, None
    for s in range(steps):
        d = _desc(src, n, div)
        kinds = {r[0] for r in records[s * n:(s + 1) * n]}
        sp = None
        if kinds & _NEEDS_STATS:
            if stats is None:
                stats = torch.empty(n * T * C.sizeof(L.AugFrameStats), dtype=torch.uint8, device=dev)
            L.check(lib.pv_augment_stats(C.byref(d), src.data_ptr(), stats.data_ptr(), stream), "pv_augment_stats")
            sp = stats.data_ptr()
        cur = bufs[s % len(bufs)]
        L.check(lib.pv_augment_apply(C.byref(d), src.data_ptr(), ops_d.data_ptr() + s * op_bytes, sp, cur.data_ptr(),
                                     stream), "pv_augment_apply")
        src, div = cur, 1
    cur._pv_keepalive = (ops_d, stats)     # device tables of the asynchronous launches
    return cur


class RandAugment:
    """RandAugment for video (reference rand_augment.py): input (T, C, H, W), or (B, T, C, H, W) with one independent
    draw per clip in clip order; uint8 or float32 CUDA tensors with any strides."""

    def __init__(self, magnitude=9, num_layers=2, prob=0.5, transform_hparas=None, sampling_type="gaussian",
                 sampling_hparas=None):
        assert sampling_type in ("gaussian", "uniform")
        sampling_hparas = sampling_hparas or RANDAUG_SAMPLING_HPARAS
        if sampling_type == "gaussian":
            assert "sampling_std" in sampling_hparas
        self.draws, self.hparas = _make_draws(OP_NAMES, magnitude, prob, RANDAUG_MAX_PARAMS, _RANDAUG_LEVEL,
                                              transform_hparas, sampling_type, sampling_hparas)
        assert 0 < num_layers <= len(self.draws), "num_layers must be in 1..%d" % len(self.draws)
        self.num_layers = num_layers

    def sample(self):
        """The ops of one clip: [(name, argument) or None for a skipped op] * num_layers."""
        return _sample_ops(self.draws, self.num_layers)

    def __call__(self, video):
        x, squeeze = _check_clips(video)
        plans = [self.sample() for _ in range(x.shape[0])]
        out = run_layers(x, plans, fill=self.hparas["fill"])
        return out[0] if squeeze else out


class AugMix:
    """AugMix for video (reference augmix.py): ``width`` chains of 1..3 (or ``depth``) ops per clip, mixed with
    Dirichlet weights and blended with the input by a Beta draw.  Input as for RandAugment."""

    def __init__(self, magnitude=3, alpha=1.0, width=3, depth=-1, transform_hparas=None, sampling_hparas=None):
        assert isinstance(magnitude, int), "magnitude must be an int"
        assert 1 <= magnitude <= MAX_LEVEL, "magnitude must be between 1 and %d inclusive" % MAX_LEVEL
        assert alpha > 0.0, "alpha must be greater than 0"
        assert width > 0, "width must be greater than 0"
        self.dirichlet = torch.distributions.dirichlet.Dirichlet(torch.tensor([alpha] * width))
        self.beta = torch.distributions.beta.Beta(alpha, alpha)
        self.draws, self.hparas = _make_draws(AUGMIX_OP_NAMES, magnitude, 1.0, AUGMIX_MAX_PARAMS, _AUGMIX_LEVEL,
                                              transform_hparas, "uniform", sampling_hparas or AUGMIX_SAMPLING_HPARAS)
        self.width = width
        self.depth, self.random_depth = (depth, False) if depth > 0 else (3, True)
        assert self.depth <= len(self.draws)

    def sample(self):
        """(mixing weights float32[width], m, [chain ops] * width) of one clip, in the reference's draw order."""
        w = self.dirichlet.sample()
        m = self.beta.sample().item()
        chains = [_sample_ops(self.draws, self.depth, self.random_depth, replacement=True) for _ in range(self.width)]
        return w, m, chains

    def __call__(self, video):
        x, squeeze = _check_clips(video)
        B = x.shape[0]
        draws = [self.sample() for _ in range(B)]
        plans = [ch for _, _, chains in draws for ch in chains]
        chains = run_layers(x, plans, src_div=self.width, fill=self.hparas["fill"])
        mix = torch.tensor([[float(v) for v in w] + [m, 1.0 - m] for w, m, _ in draws], dtype=torch.float32)
        mix_d = mix.to(x.device)
        out = torch.empty((B,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
        lib = L.load()
        d = _desc(x, B, 1)
        L.check(lib.pv_augment_mix(C.byref(d), x.data_ptr(), chains.data_ptr(), self.width, mix_d.data_ptr(),
                                   out.data_ptr(), torch.cuda.current_stream(x.device).cuda_stream), "pv_augment_mix")
        out._pv_keepalive = (chains, mix_d)
        return out[0] if squeeze else out
