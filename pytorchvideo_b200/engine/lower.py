"""Lower a PyTorchVideo-style module tree into a Plan (structural walk, no tracing).

Dispatch is by class *name* and attribute names, exactly the names the reference uses
(models/net.py, resnet.py, stem.py, head.py, slowfast.py, x3d.py, layers/convolutions.py), so the
same lowering accepts this package's own parameter-container modules and - where the reference
is importable - the reference's modules themselves (state_dict-compatible drop-in, SURVEY 8b).
"""
import weakref

import torch
import torch.nn as nn

from .. import _lib as L
from . import packing as PK
from .plan import Plan, TRef


def _t3(v):
    if isinstance(v, (tuple, list)):
        assert len(v) == 3
        return tuple(int(i) for i in v)
    return (int(v),) * 3


def _act_code(m):
    if m is None:
        return L.ACT_NONE
    n = type(m).__name__
    if n == "ReLU":
        return L.ACT_RELU
    if n == "Swish":
        return L.ACT_SWISH
    if n == "GELU":
        return L.ACT_GELU
    if n == "Sigmoid":
        return L.ACT_SIGMOID
    if n in ("HardSwish", "Hardswish"):      # the mobile blocks' wrapper and torch.nn.Hardswish
        return L.ACT_HSWISH
    if n == "Identity":
        return L.ACT_NONE
    raise NotImplementedError("activation %s has no B200 kernel" % n)


def _union_taps(convs, name):
    """Common tap box of parallel convolutions of one input (ConvReduce3D(sum) stems, the separable conv_b):
    (kernel, stride, padding, dilation, places) with places[i] the index slices of branch i inside the box.  Along
    each axis the branches with more than one tap must agree on (k, p, d); a one-tap branch sits at the box tap that
    reads the same input offset.  Anything else has no common box."""
    strides = {_t3(c.stride) for c in convs}
    if len(strides) != 1:
        raise NotImplementedError("%s: parallel convolutions with different strides %s" % (name, sorted(strides)))
    geo = [(_t3(c.kernel_size), _t3(c.padding), _t3(c.dilation)) for c in convs]
    kernel, padding, dilation = [], [], []
    for ax in range(3):
        multi = {(k[ax], p[ax], d[ax]) for k, p, d in geo if k[ax] > 1}
        if len(multi) > 1:
            raise NotImplementedError("%s: parallel convolutions with different taps along axis %d" % (name, ax))
        if multi:
            k, p, d = multi.pop()
        else:
            pads = {p[ax] for _, p, _ in geo}
            if len(pads) != 1:
                raise NotImplementedError("%s: one-tap branches with different paddings along axis %d" % (name, ax))
            k, p, d = 1, pads.pop(), 1
        kernel.append(k)
        padding.append(p)
        dilation.append(d)
    places = []
    for kb, pb, _ in geo:
        sl = []
        for ax in range(3):
            if kb[ax] > 1:
                sl.append(slice(0, kernel[ax]))
                continue
            j, r = divmod(padding[ax] - pb[ax], dilation[ax])     # box tap j reads input offset j * d - p = -pb
            if r or not 0 <= j < kernel[ax]:
                raise NotImplementedError("%s: branch padding is not centre-consistent along axis %d" % (name, ax))
            sl.append(slice(j, j + 1))
        places.append(tuple(sl))
    return tuple(kernel), strides.pop(), tuple(padding), tuple(dilation), places


def _is_bn(m):
    return isinstance(m, nn.modules.batchnorm._BatchNorm) or type(m).__name__.startswith("NaiveSyncBatchNorm")


class Lowering:
    def __init__(self, plan: Plan, extra=()):
        self.p = plan
        self.extra = tuple(extra)     # non-tensor forward arguments of the root module (thw_shape)
        self.aux_out = None           # host-side second result of the root module (pooled thw)
        self.fuse_rows = False        # Linear -> ReLU as one launch (models/embedding.py EmbeddingChain)

    # ---- leaf helpers --------------------------------------------------------------------
    def conv(self, x: TRef, conv: nn.Conv3d, bn=None, act=None, residual=None, name="conv", se_sums=False, addend=None):
        if type(conv).__name__ == "Conv2plus1d":
            if addend is not None:
                raise NotImplementedError("%s: Conv2plus1d takes no addend" % name)
            return self.conv2plus1d(x, conv, bn, act, residual, name)
        if not isinstance(conv, nn.Conv3d):
            raise NotImplementedError("%s: conv module %s unsupported" % (name, type(conv).__name__))
        if isinstance(conv.padding, str):
            raise NotImplementedError("string padding unsupported")
        if conv.padding_mode != "zeros":
            raise NotImplementedError("padding_mode %s unsupported" % conv.padding_mode)
        if bn is not None and not _is_bn(bn):
            raise NotImplementedError("%s: norm %s unsupported (BatchNorm only)" % (name, type(bn).__name__))
        return self.p.emit_conv(x, conv.weight, conv.bias, bn, _t3(conv.stride), _t3(conv.padding),
                                _t3(conv.dilation), conv.groups, _act_code(act), residual, name, se_sums=se_sums,
                                addend=addend)

    def conv2plus1d(self, x, m, bn, act, residual, name):
        # layers/convolutions.py:232-237: conv_t -> norm -> activation -> conv_xy, or conv_xy first when
        # conv_xy_first is set (the flag only swaps the two convolutions; norm/activation stay in between)
        first, second = ("conv_xy", "conv_t") if getattr(m, "conv_xy_first", False) else ("conv_t", "conv_xy")
        h = self.conv(x, getattr(m, first), getattr(m, "norm", None), getattr(m, "activation", None), None,
                      name + "." + first)
        return self.conv(h, getattr(m, second), bn, act, residual, name + "." + second)

    def lower_Conv2plus1d(self, m, x, name):
        return self.conv2plus1d(x, m, None, None, None, name)

    def lower_Conv3d(self, m, x, name):
        return self.conv(x, m, None, None, None, name or "conv")

    def lower_ConvReduce3D(self, m, x, name):
        # layers/convolutions.py:77-85: parallel convolutions of one input, summed (stack().sum(0)) or
        # concatenated along channels.  sum: every conv after the first takes the running sum as the fused
        # residual of its epilogue (fp32 add on the accumulator); cat: producers write channel slices.
        outs = []
        acc = None
        for i, c in enumerate(m.convs):
            if m.reduction_method == "sum":
                acc = self.conv(x, c, None, None, acc, "%s.convs.%d" % (name, i))
            else:
                outs.append(self.conv(x, c, None, None, None, "%s.convs.%d" % (name, i)))
        if m.reduction_method == "sum":
            return acc
        for o in outs[:-1]:
            if o.C != o.Cp:
                raise NotImplementedError("ConvReduce3D(cat): out_channels must be a multiple of 8 for the fused concat")
        return self.p.concat_channels(outs) if len(outs) > 1 else outs[0]

    def lower_Swish(self, m, x, name):
        self.p.materialize_input(x)
        return self.p.emit_act(x, L.ACT_SWISH, name or "swish")

    def lower_ReLU(self, m, x, name):
        self.p.materialize_input(x)
        return self.p.emit_act(x, L.ACT_RELU, name or "relu")

    def lower_SqueezeExcitation(self, m, x, name):
        blk = _se_block(m, name or "se")
        if type(blk[1]).__name__ != "ReLU" or type(blk[3]).__name__ != "Sigmoid":
            raise NotImplementedError("SqueezeExcitation variant unsupported")
        self.p.materialize_input(x)
        return self.p.emit_se_scale_act(x, blk[0].weight, blk[0].bias, blk[2].weight, blk[2].bias, L.ACT_NONE,
                                        name or "se")

    def pool(self, x, m, name="pool"):
        n = type(m).__name__
        if n == "MaxPool3d":
            if _t3(m.dilation) != (1, 1, 1) or m.ceil_mode:
                raise NotImplementedError("MaxPool3d dilation/ceil_mode unsupported")
            k = _t3(m.kernel_size)
            s = _t3(m.stride if m.stride is not None else m.kernel_size)
            return self.p.emit_pool(x, L.POOL_MAX, k, s, _t3(m.padding), name)
        if n == "AvgPool3d":
            if m.ceil_mode or not m.count_include_pad or m.divisor_override is not None:
                raise NotImplementedError("AvgPool3d options unsupported")
            k = _t3(m.kernel_size)
            s = _t3(m.stride if m.stride is not None else m.kernel_size)
            return self.p.emit_pool(x, L.POOL_AVG, k, s, _t3(m.padding), name)
        if n == "AdaptiveAvgPool3d":
            osz = _t3(m.output_size)
            if osz != (1, 1, 1):
                raise NotImplementedError("AdaptiveAvgPool3d output_size %s unsupported" % (osz,))
            k = (x.T, x.H, x.W)
            return self.p.emit_pool(x, L.POOL_AVG, k, k, (0, 0, 0), name)
        if n == "Identity":
            return x
        raise NotImplementedError("pool module %s unsupported" % n)

    # ---- blocks --------------------------------------------------------------------------
    def lower(self, m, x, name=""):
        n = type(m).__name__
        fn = getattr(self, "lower_" + n, None)
        if fn is None:
            raise NotImplementedError("no B200 lowering for module %s (%s)" % (n, name))
        return fn(m, x, name)

    def lower_Identity(self, m, x, name):
        return x

    def lower_Dropout(self, m, x, name):
        return x   # eval mode

    def lower_MaxPool3d(self, m, x, name):
        return self.pool(x, m, name)

    lower_AvgPool3d = lower_MaxPool3d
    lower_AdaptiveAvgPool3d = lower_MaxPool3d

    def lower_Net(self, m, x, name):
        # models/net.py:41-44
        for i, blk in enumerate(m.blocks):
            x = self.lower(blk, x, "%sblocks.%d" % (name + "." if name else "", i))
        return x

    def lower_Sequential(self, m, x, name):
        mods = list(m)
        i = 0
        while i < len(mods):
            # Linear -> BatchNorm (which has no lowering of its own) always fuses; inside the embedding path of the
            # self-supervised models (``fuse_rows``) a Linear -> ReLU fuses as well
            if isinstance(mods[i], nn.Linear) and isinstance(x, TRef) and (
                    self.fuse_rows or (i + 1 < len(mods) and _is_bn(mods[i + 1]))):
                x, i = _lower_linear_chain(self, mods, i, x, name)
                continue
            x = self.lower(mods[i], x, "%s.%d" % (name, i))
            i += 1
        return x

    def lower_ResNetBasicStem(self, m, x, name, addend=None):
        # models/stem.py:252-260: conv -> norm -> activation -> pool
        pool = getattr(m, "pool", None)
        if addend is not None and pool is not None:
            # the addend is constant over (h, w) and max pooling pads with -inf, so maxpool(y) + a == maxpool(y + a)
            # for a pool that does not mix frames: the add moves into the conv's epilogue
            if type(pool).__name__ != "MaxPool3d" or _t3(pool.kernel_size)[0] != 1 or \
                    _t3(pool.stride if pool.stride is not None else pool.kernel_size)[0] != 1 or _t3(pool.padding)[0] != 0:
                raise NotImplementedError("%s: an audio fusion after the stem needs a spatial-only MaxPool3d" % name)
        if type(m.conv).__name__ == "ConvReduce3D":
            x = self.conv_reduce_sum(x, m.conv, m.norm, m.activation, name + ".conv", addend)
        else:
            x = self.conv(x, m.conv, m.norm, m.activation, None, name + ".conv", addend=addend)
        if pool is not None:
            x = self.pool(x, pool, name + ".pool")
        return x

    def conv_reduce_sum(self, x, m, bn, act, name, addend=None):
        """The acoustic stem's ConvReduce3D (stem.py:179-192): a (kt,1,1) and a (1,kh,kw) convolution of one input,
        summed, as ONE convolution whose kernel is the sum of both embedded in their common (kt,kh,kw) box (exact;
        the network input can also feed only one window-mode stem convolution)."""
        if m.reduction_method != "sum":
            raise NotImplementedError("%s: ConvReduce3D(cat) in a stem is unsupported" % name)
        convs = list(m.convs)
        for c in convs:
            if type(c) is not nn.Conv3d or isinstance(c.padding, str) or c.padding_mode != "zeros":
                raise NotImplementedError("%s: ConvReduce3D branches must be zero-padded Conv3d" % name)
        if len({c.groups for c in convs}) != 1:
            raise NotImplementedError("%s: ConvReduce3D branches with different groups" % name)
        kernel, stride, padding, dilation, places = _union_taps(convs, name)
        c0 = convs[0]
        w = torch.zeros((c0.out_channels, c0.in_channels // c0.groups) + kernel, dtype=torch.float64)
        for c, sl in zip(convs, places):
            w[(slice(None), slice(None)) + sl] += c.weight.detach().double().cpu()
        biases = [c.bias for c in convs if c.bias is not None]
        bias = sum(b.detach().double().cpu() for b in biases).float() if biases else None
        if bn is not None and not _is_bn(bn):
            raise NotImplementedError("%s: norm %s unsupported (BatchNorm only)" % (name, type(bn).__name__))
        return self.p.emit_conv(x, w.float(), bias, bn, stride, padding, dilation, c0.groups, _act_code(act), None,
                                name, addend=addend)

    def lower_ResStage(self, m, x, name, addend=None):
        n = len(m.res_blocks)
        for i, blk in enumerate(m.res_blocks):
            bname = "%s.res_blocks.%d" % (name, i)
            if addend is not None and i == n - 1:
                if type(blk).__name__ != "ResBlock":
                    raise NotImplementedError("%s: an audio fusion needs a ResBlock at the end of the stage" % bname)
                x = self.lower_ResBlock(blk, x, bname, addend)
            else:
                x = self.lower(blk, x, bname)
        return x

    def _fusable_bottleneck(self, m, x):
        """ResBlock whose whole body runs as ONE launch of the fused narrow-pathway kernel (csrc/pv_fastblock.cu):
        plain Conv3d / BatchNorm / ReLU bottleneck with a (kt,1,1) conv_a, a dense (1,3,3) conv_b of stride
        (1,s,s) and an inner width of 8 / 16 / 32 channels (the SlowFast Fast pathway, res2-res4)."""
        import ctypes as C_
        p = self.p
        if p.dt != L.PV_F16:
            return False
        b = m.branch2
        if type(b).__name__ != "BottleneckBlock" or not isinstance(x, TRef):
            return False
        convs = (b.conv_a, b.conv_b, b.conv_c) + ((m.branch1_conv,) if m.branch1_conv is not None else ())
        for c in convs:
            if type(c) is not nn.Conv3d or c.groups != 1 or _t3(c.dilation) != (1, 1, 1) or c.padding_mode != "zeros" \
                    or isinstance(c.padding, str):
                return False
        for n_ in (b.norm_a, b.norm_b, b.norm_c):
            if n_ is None or not _is_bn(n_):
                return False
        if type(b.act_a).__name__ != "ReLU" or type(b.act_b).__name__ != "ReLU":
            return False
        if m.activation is not None and type(m.activation).__name__ not in ("ReLU", "Identity"):
            return False
        ka, kb, kc = _t3(b.conv_a.kernel_size), _t3(b.conv_b.kernel_size), _t3(b.conv_c.kernel_size)
        if ka[1:] != (1, 1) or ka[0] not in (1, 3) or _t3(b.conv_a.stride) != (1, 1, 1) or _t3(b.conv_a.padding) != (ka[0] // 2, 0, 0):
            return False
        sb = _t3(b.conv_b.stride)
        if kb != (1, 3, 3) or sb[0] != 1 or sb[1] != sb[2] or sb[1] not in (1, 2) or _t3(b.conv_b.padding) != (0, 1, 1):
            return False
        if kc != (1, 1, 1) or _t3(b.conv_c.stride) != (1, 1, 1) or _t3(b.conv_c.padding) != (0, 0, 0):
            return False
        if b.conv_a.in_channels != x.C or x.C != x.Cp:      # (a 3-channel network input is padded to 4: not this kernel)
            return False
        if m.branch1_conv is not None:
            c1 = m.branch1_conv
            if _t3(c1.kernel_size) != (1, 1, 1) or _t3(c1.stride) != (1, sb[1], sb[1]) or _t3(c1.padding) != (0, 0, 0):
                return False
            n1 = getattr(m, "branch1_norm", None)
            if n1 is not None and not _is_bn(n1):
                return False
        act = L.ACT_RELU if (m.activation is not None and type(m.activation).__name__ == "ReLU") else L.ACT_NONE
        d = p.fused_bottleneck_desc(x, x.Cp, b.conv_a.out_channels, b.conv_c.out_channels, ka[0], sb[1],
                                    m.branch1_conv is not None, act)
        return bool(p.lib.pv_bottleneck_fused_supported(C_.byref(d)))

    def lower_ResBlock(self, m, x, name, addend=None):
        # models/resnet.py:1179-1189; branch_fusion is x + y for every builder in scope.  The fused narrow-block
        # kernel has no addend: a block that takes one runs as separate convolutions.
        if addend is None and self._fusable_bottleneck(m, x):
            b = m.branch2
            act = L.ACT_RELU if (m.activation is not None and type(m.activation).__name__ == "ReLU") else L.ACT_NONE
            return self.p.emit_bottleneck_fused(x, b.conv_a, b.norm_a, b.conv_b, b.norm_b, b.conv_c, b.norm_c,
                                                m.branch1_conv, getattr(m, "branch1_norm", None), act, name + ".fused")
        if m.branch1_conv is not None:
            shortcut = self.conv(x, m.branch1_conv, getattr(m, "branch1_norm", None), None, None, name + ".branch1")
        else:
            shortcut = x
        return self.bottleneck(m.branch2, x, shortcut, m.activation, name + ".branch2", addend)

    def lower_BottleneckBlock(self, m, x, name):
        return self.bottleneck(m, x, None, None, name)

    lower_SeparableBottleneckBlock = lower_BottleneckBlock

    def bottleneck(self, m, x, shortcut, final_act, name, addend=None):
        # models/resnet.py:1345-1365 with the block's residual add + activation fused into conv_c
        if type(m).__name__ == "SeparableBottleneckBlock":
            return self.separable_bottleneck(m, x, shortcut, final_act, name, addend)
        if type(m).__name__ != "BottleneckBlock":
            raise NotImplementedError("branch2 module %s unsupported" % type(m).__name__)
        h = self.conv(x, m.conv_a, m.norm_a, m.act_a, None, name + ".conv_a")
        norm_b, se = m.norm_b, None
        if isinstance(norm_b, nn.Sequential):      # X3D: Sequential(BN|Identity, SE|Identity), models/x3d.py:199-208
            assert len(norm_b) == 2
            se = norm_b[1] if type(norm_b[1]).__name__ == "SqueezeExcitation" else None
            if se is None and type(norm_b[1]).__name__ != "Identity":
                raise NotImplementedError("norm_b[1] %s unsupported" % type(norm_b[1]).__name__)
            norm_b = norm_b[0] if _is_bn(norm_b[0]) else None
        if se is None:
            h = self.conv(h, m.conv_b, norm_b, m.act_b, None, name + ".conv_b")
        else:
            h = self.conv(h, m.conv_b, norm_b, None, None, name + ".conv_b", se_sums=True)
            blk = se.block
            if type(blk[1]).__name__ != "ReLU" or type(blk[3]).__name__ != "Sigmoid":
                raise NotImplementedError("SqueezeExcitation variant unsupported")
            h = self.p.emit_se_scale_act(h, blk[0].weight, blk[0].bias, blk[2].weight, blk[2].bias,
                                         _act_code(m.act_b), name + ".se")
        return self.conv(h, m.conv_c, m.norm_c, final_act, shortcut, name + ".conv_c", addend=addend)

    def separable_bottleneck(self, m, x, shortcut, final_act, name, addend=None):
        """SeparableBottleneckBlock (models/resnet.py:1257-1285).  Both conv_b branches run as ONE convolution over
        the union of their taps (zero where a branch has none), output channels [branch 0 | branch 1], each with its
        own folded norm; "cat" is that output, "sum" feeds conv_c with its weight repeated along C_in,
        conv_c(a + b) = [W_c | W_c] . [a ; b], so the sum is never materialised."""
        h = x
        if m.conv_a is not None:
            h = self.conv(x, m.conv_a, m.norm_a, m.act_a, None, name + ".conv_a")
        convs, norms, acts = list(m.conv_b), list(m.norm_b), list(m.act_b)
        for c in convs:
            if type(c) is not nn.Conv3d or isinstance(c.padding, str) or c.padding_mode != "zeros":
                raise NotImplementedError("%s.conv_b: branches must be zero-padded Conv3d" % name)
            if c.in_channels != h.C:
                raise RuntimeError("conv %s.conv_b expects %d input channels, got %d" % (name, c.in_channels, h.C))
        for n_ in norms:
            if n_ is not None and not _is_bn(n_):
                raise NotImplementedError("%s.norm_b: norm %s unsupported (BatchNorm only)" % (name, type(n_).__name__))
        act_names = {None if a is None else type(a).__name__ for a in acts}
        if len(act_names) != 1:
            raise NotImplementedError("%s.act_b: branches with different activations %s" % (name, sorted(map(str, act_names))))
        kernel, stride, padding, dilation, places = _union_taps(convs, name + ".conv_b")
        dense = [PK.expand_grouped_dense(c.weight, c.groups) if c.groups != 1 else c.weight.detach().cpu() for c in convs]
        rows = [c.out_channels for c in convs]
        w = torch.zeros((sum(rows), h.C) + kernel, dtype=dense[0].dtype)
        o = 0
        for wd, r, sl in zip(dense, rows, places):
            w[(slice(o, o + r), slice(None)) + sl] = wd
            o += r
        folded = [PK.fold_bn(c.bias, n_, c.out_channels, c.out_channels) for c, n_ in zip(convs, norms)]
        folded = (torch.cat([f[0] for f in folded]), torch.cat([f[1] for f in folded]))
        h = self.p.emit_conv(h, w, None, None, stride, padding, dilation, 1, _act_code(acts[0]), None,
                             name + ".conv_b", folded=folded)
        cc = m.conv_c
        if m.reduce_method == "sum":
            if len(set(rows)) != 1:
                raise RuntimeError("%s: summed conv_b branches need equal widths, got %s" % (name, rows))
            if type(cc) is not nn.Conv3d or cc.groups != 1:
                raise NotImplementedError("%s.conv_c: Conv3d with groups 1 expected" % name)
            if cc.in_channels != rows[0]:
                raise RuntimeError("conv %s.conv_c expects %d input channels, got %d" % (name, cc.in_channels, rows[0]))
            wc = torch.cat([cc.weight.detach().cpu()] * len(rows), 1)
            return self.p.emit_conv(h, wc, cc.bias, m.norm_c, _t3(cc.stride), _t3(cc.padding), _t3(cc.dilation), 1,
                                    _act_code(final_act), shortcut, name + ".conv_c", addend=addend)
        return self.conv(h, cc, m.norm_c, final_act, shortcut, name + ".conv_c", addend=addend)

    # head widths of the Non-local attention core (csrc/pv_attention.cu routing): softmax also runs on the MViT
    # kernels' 32 / 96, the linear ("dot_product") mode only on the widths of csrc/pv_attention_wide.cu
    _NL_DIMS = {"softmax": (32, 64, 96, 128, 256, 512), "dot_product": (64, 128, 256, 512)}

    def lower_NonLocal(self, m, x, name):
        # layers/nonlocal_net.py:55-94: theta from x, phi / g from pool(x), one single-head attention of width
        # dim_inner, conv_out (+ norm) with x as the fused residual; no activation
        name = name or "nonlocal"
        convs = (m.conv_theta, m.conv_phi, m.conv_g, m.conv_out)
        for cn, c in zip(("conv_theta", "conv_phi", "conv_g", "conv_out"), convs):
            if not isinstance(c, nn.Conv3d) or _t3(c.kernel_size) != (1, 1, 1) or _t3(c.stride) != (1, 1, 1) \
                    or isinstance(c.padding, str) or _t3(c.padding) != (0, 0, 0) or _t3(c.dilation) != (1, 1, 1) \
                    or c.groups != 1:
                raise NotImplementedError("%s.%s: NonLocal needs 1x1x1 convolutions of stride 1, groups 1" % (name, cn))
        if m.norm is not None and not _is_bn(m.norm):
            raise NotImplementedError("%s: norm %s unsupported (BatchNorm only)" % (name, type(m.norm).__name__))
        if m.instantiation not in self._NL_DIMS:
            raise NotImplementedError("%s: instantiation %r unsupported" % (name, m.instantiation))
        di = m.conv_theta.out_channels
        if di not in self._NL_DIMS[m.instantiation]:
            raise NotImplementedError("%s: dim_inner %d unsupported for %s (supported: %s)" % (
                name, di, m.instantiation, self._NL_DIMS[m.instantiation]))
        if m.conv_theta.in_channels != x.C:
            raise RuntimeError("conv %s.conv_theta expects %d input channels, got %d" % (name, m.conv_theta.in_channels, x.C))

        def fused(cs):
            w = torch.cat([c.weight for c in cs], 0)
            if all(c.bias is None for c in cs):
                return w, None
            return w, torch.cat([c.bias if c.bias is not None else torch.zeros(c.out_channels) for c in cs], 0)

        p = self.p
        if m.pool is not None:
            w, b = fused((m.conv_theta,))
            theta = p.emit_conv(x, w, b, None, (1, 1, 1), (0, 0, 0), (1, 1, 1), 1, L.ACT_NONE, None, name + ".conv_theta")
            xp = self.pool(x, m.pool, name + ".pool")
            w, b = fused((m.conv_phi, m.conv_g))
            pg = p.emit_conv(xp, w, b, None, (1, 1, 1), (0, 0, 0), (1, 1, 1), 1, L.ACT_NONE, None, name + ".conv_phi_g")
            phi, g = PL.channel_slice(pg, 0, di), PL.channel_slice(pg, di, di)
        else:
            w, b = fused((m.conv_theta, m.conv_phi, m.conv_g))
            tpg = p.emit_conv(x, w, b, None, (1, 1, 1), (0, 0, 0), (1, 1, 1), 1, L.ACT_NONE, None,
                              name + ".conv_theta_phi_g")
            theta, phi, g = (PL.channel_slice(tpg, i * di, di) for i in range(3))
        if m.instantiation == "softmax":
            o = PL.emit_attention(p, theta, phi, g, 1, di ** -0.5, False, name + ".attention")
        else:
            o = PL.emit_attention(p, theta, phi, g, 1, 1.0, False, name + ".attention", normalize=1)
        # the attention output is token-major [N][T*H*W][dim_inner]: the same rows as x, so give it x's grid back
        o = TRef(o.buf, x.N, x.T, x.H, x.W, o.C, Cp=o.Cp, ch_off=o.ch_off, row_stride=o.row_stride)
        return self.conv(o, m.conv_out, m.norm, None, x, name + ".conv_out")

    def lower_MultiPathWayWithFuse(self, m, x, name):
        # models/net.py:107-122
        assert isinstance(x, list), "input for MultiPathWayWithFuse needs to be a list of tensors"
        if type(m.multipathway_fusion).__name__ == "FuseAudioToFastSlow":
            return self.audio_fused_stage(m, x, name)
        out = list(x)
        # the pathways are independent until the fusion: each gets its own lane (CUDA stream / graph branch)
        for i, blk in enumerate(m.multipathway_blocks):
            if blk is not None:
                self.p.lane = i
                out[i] = self.lower(blk, x[i], "%s.multipathway_blocks.%d" % (name, i))
        self.p.lane = 0
        if m.multipathway_fusion is not None:
            out = self.lower(m.multipathway_fusion, out, name + ".multipathway_fusion")
        return out

    def lower_FuseFastToSlow(self, m, x, name):
        # models/slowfast.py:720-729; the concat is fused away (both producers write into one buffer)
        x_s, x_f = x[0], x[1]
        self.p.lane = 1        # the lateral conv reads the Fast tensor: keep it on the Fast lane, the Slow lane only
        fuse = self.conv(x_f, m.conv_fast_to_slow, m.norm, m.activation, None, name + ".conv_fast_to_slow")
        self.p.lane = 0        # waits for it where the next Slow stage reads the concat buffer
        return [self.p.concat_channels([x_s, fuse]), x_f]

    def audio_fused_stage(self, m, x, name):
        """One AVSlowFast stage: the pathways, then FuseAudioToFastSlow (models/audio_visual_slowfast.py:406-418),
        [fuse_a + cat(x_s, conv_f2s(x_f)), x_f, x_a].  Both writers of the concat buffer - the Slow pathway's last
        convolution and the Fast->Slow convolution - add fuse_a in their epilogues, so neither the concat nor the add
        is a pass of its own.  Emission order: the audio pathway and the fuse_a chain (lane 2) come first, so every
        op that takes fuse_a is emitted after its writer and waits for it across lanes (Plan._schedule)."""
        if len(x) != 3:
            raise RuntimeError("FuseAudioToFastSlow takes [slow, fast, audio] pathways, got %d" % len(x))
        p = self.p
        blocks, fusion = m.multipathway_blocks, m.multipathway_fusion
        bname = "%s.multipathway_blocks.%%d" % name
        fname = name + ".multipathway_fusion"
        out = list(x)
        p.lane = 2
        if blocks[2] is not None:
            out[2] = self.lower(blocks[2], x[2], bname % 2)
        xa = out[2]
        a = p.emit_pool(xa, L.POOL_AVG, (1, 1, xa.W), (1, 1, xa.W), (0, 0, 0), fname + ".mean")   # mean over F
        a = self.conv_chain(fusion.block_audio_to_fastslow, a, fname + ".block_audio_to_fastslow")
        p.lane = 0
        slow = blocks[0]
        sn = type(slow).__name__
        if sn == "ResStage":
            out[0] = self.lower_ResStage(slow, x[0], bname % 0, addend=(a, 0))
        elif sn == "ResNetBasicStem":
            out[0] = self.lower_ResNetBasicStem(slow, x[0], bname % 0, addend=(a, 0))
        else:
            raise NotImplementedError("%s: Slow pathway block %s cannot take the audio fusion" % (name, sn))
        p.lane = 1
        if blocks[1] is not None:
            out[1] = self.lower(blocks[1], x[1], bname % 1)
        x_s = out[0]
        f2s = list(fusion.block_fast_to_slow)
        c_fuse = f2s[0].out_channels if f2s and isinstance(f2s[0], nn.Conv3d) else 0
        if a.C != x_s.C + c_fuse:
            raise RuntimeError("%s: audio fusion has %d channels, the Slow concat %d" % (fname, a.C, x_s.C + c_fuse))
        if x_s.C != x_s.Cp:
            raise NotImplementedError("%s: Slow pathway width %d is not a multiple of 8" % (fname, x_s.C))
        fuse = self.conv_chain(fusion.block_fast_to_slow, out[1], fname + ".block_fast_to_slow", addend=(a, x_s.Cp))
        p.lane = 0
        return [p.concat_channels([x_s, fuse]), out[1], out[2]]

    def conv_chain(self, seq, x, name, addend=None):
        """nn.Sequential of Conv3d [+ BatchNorm] [+ activation] groups (the FuseAudioToFastSlow blocks); the addend
        goes to the last convolution."""
        mods = list(seq)
        groups, i = [], 0
        while i < len(mods):
            c = mods[i]
            if not isinstance(c, nn.Conv3d):
                raise NotImplementedError("%s.%d: %s unsupported here (Conv3d expected)" % (name, i, type(c).__name__))
            j, bn, act = i + 1, None, None
            if j < len(mods) and _is_bn(mods[j]):
                bn, j = mods[j], j + 1
            if j < len(mods) and not isinstance(mods[j], nn.Conv3d) and not _is_bn(mods[j]):
                act, j = mods[j], j + 1
            groups.append((i, c, bn, act))
            i = j
        if not groups:
            raise NotImplementedError("%s: empty convolution chain" % name)
        for g, (i, c, bn, act) in enumerate(groups):
            x = self.conv(x, c, bn, act, None, "%s.%d" % (name, i), addend=addend if g == len(groups) - 1 else None)
        return x

    def lower_PoolConcatPathway(self, m, x, name):
        # models/slowfast.py:608-620
        outs = []
        for i, xi in enumerate(x):
            if xi is None:
                continue
            if m.pool is not None and m.pool[i] is not None:
                self.p.lane = i
                xi = self.pool(xi, m.pool[i], "%s.pool.%d" % (name, i))
                self.p.lane = 0
            outs.append(xi)
        cat = self.p.concat_channels(outs) if len(outs) > 1 else outs[0]
        return [cat] if getattr(m, "retain_list", False) else cat

    def lower_ProjectedPool(self, m, x, name):
        # models/x3d.py:791-806
        x = self.conv(x, m.pre_conv, m.pre_norm, m.pre_act, None, name + ".pre_conv")
        x = self.pool(x, m.pool, name + ".pool")
        return self.conv(x, m.post_conv, m.post_norm, m.post_act, None, name + ".post_conv")

    def lower_DetectionBBoxNetwork(self, m, x, name):
        # models/net.py:62-74: features = model(x); out = detection_head(features, bboxes); out.view(K, -1)
        feats = self.lower(m.model, x[0] if len(x) == 2 else list(x[:-1]), (name + "." if name else "") + "model")
        return self.lower_ResNetRoIHead(m.detection_head, [feats, x[-1]], (name + "." if name else "") + "detection_head")

    def lower_ResNetRoIHead(self, m, x, name):
        # models/head.py:441-482
        if len(x) != 2:
            raise RuntimeError("ResNetRoIHead.forward(x, bboxes) takes one feature tensor and the boxes")
        x, boxes = x
        if isinstance(x, list):
            raise RuntimeError("ResNetRoIHead expects ONE feature tensor (PoolConcatPathway(retain_list=False))")
        name = name or "head"
        if getattr(m, "pool", None) is not None:
            x = self.pool(x, m.pool, name + ".pool")
        roi = getattr(m, "roi_layer", None)
        if roi is not None:
            if type(roi).__name__ != "RoIAlign":
                raise NotImplementedError("roi layer %s unsupported (RoIAlign only)" % type(roi).__name__)
            if getattr(roi, "aligned", False):
                raise NotImplementedError("RoIAlign(aligned=True) unsupported")
            osz = roi.output_size
            osz = (osz, osz) if isinstance(osz, int) else tuple(osz)
            x = self.p.emit_roi_align(x, boxes, osz, roi.spatial_scale, roi.sampling_ratio, name + ".roi_layer")
            ps = getattr(m, "pool_spatial", None)
            if ps is not None:
                pn = type(ps).__name__
                if pn not in ("MaxPool2d", "AvgPool2d"):
                    raise NotImplementedError("pool_spatial %s unsupported" % pn)
                k2 = ps.kernel_size if isinstance(ps.kernel_size, (tuple, list)) else (ps.kernel_size,) * 2
                s2 = ps.stride if isinstance(ps.stride, (tuple, list)) else (ps.stride,) * 2
                p2 = ps.padding if isinstance(ps.padding, (tuple, list)) else (ps.padding,) * 2
                if pn == "MaxPool2d" and (ps.dilation not in (1, (1, 1)) or ps.ceil_mode):
                    raise NotImplementedError("MaxPool2d dilation/ceil_mode unsupported")
                if pn == "AvgPool2d" and (ps.ceil_mode or not ps.count_include_pad or ps.divisor_override is not None):
                    raise NotImplementedError("AvgPool2d options unsupported")
                x = self.p.emit_pool(x, L.POOL_MAX if pn == "MaxPool2d" else L.POOL_AVG, (1,) + tuple(k2), (1,) + tuple(s2),
                                     (0,) + tuple(p2), name + ".pool_spatial")
        proj = m.proj
        if not isinstance(proj, nn.Linear):
            raise NotImplementedError("head proj %s unsupported" % type(proj).__name__)
        act = getattr(m, "activation", None)
        an = None if act is None else type(act).__name__
        if an not in (None, "Sigmoid", "ReLU", "Identity"):
            raise NotImplementedError("RoI head activation %s unsupported" % an)
        w = proj.weight.reshape(proj.out_features, proj.in_features, 1, 1, 1)
        x = self.p.emit_conv(x, w, proj.bias, None, (1, 1, 1), (0, 0, 0), (1, 1, 1), 1,
                             L.ACT_RELU if an == "ReLU" else L.ACT_NONE, None, name + ".proj")
        if an == "Sigmoid":
            x = self.p.emit_act(x, L.ACT_SIGMOID, name + ".activation")
        if getattr(m, "output_pool", None) is not None:
            return self.p.emit_head_reduce(x, False, name + ".output_pool")       # AdaptiveAvgPool3d(1) + view(K, -1)
        return self.p.emit_to_ncdhw(x, name + ".to_ncdhw")

    def lower_ResNetBasicHead(self, m, x, name):
        # models/head.py:371-391
        pool = getattr(m, "pool", None)
        if pool is not None:
            x = self.lower(pool, x, name + ".pool") if type(pool).__name__ == "ProjectedPool" else self.pool(x, pool, name + ".pool")
        proj = m.proj
        if proj is None:
            return _lower_headless(self, m, x, name)
        if not isinstance(proj, nn.Linear):
            raise NotImplementedError("head proj %s unsupported" % type(proj).__name__)
        w = proj.weight.reshape(proj.out_features, proj.in_features, 1, 1, 1)
        x = self.p.emit_conv(x, w, proj.bias, None, (1, 1, 1), (0, 0, 0), (1, 1, 1), 1, L.ACT_NONE, None, name + ".proj")
        act = getattr(m, "activation", None)
        softmax = False
        if act is not None:
            an = type(act).__name__
            if an == "Softmax":
                if act.dim != 1:
                    raise NotImplementedError("head softmax dim != 1")
                softmax = True
            elif an == "Sigmoid":
                x = self.p.emit_act(x, L.ACT_SIGMOID, name + ".activation")
            else:
                raise NotImplementedError("head activation %s unsupported" % an)
        if getattr(m, "output_pool", None) is not None:
            return self.p.emit_head_reduce(x, softmax, name + ".output_pool")
        if softmax:
            raise NotImplementedError("head softmax without output_pool unsupported")
        return self.p.emit_to_ncdhw(x, name + ".to_ncdhw")


class CompiledModel:
    """A frozen (model, input shapes) plan: static input/output buffers + one CUDA graph.

    Inputs are 5-D clips (B, C, T, H, W) - or, for the MViT layer modules, token tensors (B, N, C) / (B, C).
    ``extra`` carries non-tensor forward arguments (the ``thw_shape`` of MultiScaleBlock / MultiScaleAttention);
    a lowering handler may leave a second, host-side result in ``Lowering.aux_out`` (the pooled thw)."""

    def __init__(self, model, example_inputs, dtype="f16", use_graph=True, extra=()):
        L.require_device()
        multi = isinstance(example_inputs, (list, tuple))
        ins = list(example_inputs) if multi else [example_inputs]
        raw = _raw_inputs(model, ins)
        self.mask_slots = _mask_slots(ins, extra)
        image = _image_root(model, ins)
        for i, t in enumerate(ins):
            if i not in raw and i not in self.mask_slots and t.dim() not in (2, 3, 5) and not image:
                raise RuntimeError("expected a 5-D (B, C, T, H, W) clip or a (B, N, C) token tensor, got %s" % (tuple(t.shape),))
        device = ins[0].device
        if device.type != "cuda":
            raise RuntimeError("pytorchvideo_b200 has no CPU path: inputs must be CUDA tensors")
        dt = {"f16": L.PV_F16, "f32": L.PV_F32}[dtype]
        self.multi = multi
        self.plan = Plan(device, dt)
        self.static_in = [torch.empty(t.shape, dtype=torch.uint8 if i in self.mask_slots else
                                      t.dtype if (t.dtype in (torch.float16, torch.float32) and i not in raw)
                                      else torch.float32, device=device) for i, t in enumerate(ins)]
        low = Lowering(self.plan, extra)
        xs = [self.plan.raw_input(s) if i in raw else PL.MaskRef(s.shape[0], s.shape[1], tensor=s) if i in self.mask_slots
              else _emit_input(self.plan, s) for i, s in enumerate(self.static_in)]
        out = low.lower(model, _root_input(xs, ins, extra) if _masked_root(extra) else (xs if multi else xs[0]), "")
        out = _emit_output(self.plan, out, tokens=ins[0].dim() not in (4, 5))
        self.out_buf, self.out_shape = out
        self.aux = low.aux_out
        self.plan.finalize()
        self.graph = None
        self.use_graph = use_graph
        self.key = tuple((tuple(t.shape), t.dtype) for t in ins)

    def _capture(self):
        dev = self.plan.device
        stream = torch.cuda.Stream(device=dev)
        stream.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(stream):
            self.plan.run(stream.cuda_stream)       # warm-up (also sets func attributes outside capture)
        torch.cuda.current_stream(dev).wait_stream(stream)
        torch.cuda.synchronize(dev)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            self.plan.run(torch.cuda.current_stream(dev).cuda_stream)
        self.graph = g

    def pipeline(self, depth=2):
        """Double-buffered host-in / host-out serving loop (engine/pipeline.py)."""
        from .pipeline import ClipPipeline
        return ClipPipeline(self, depth)

    def output_view(self):
        return self.out_buf.tensor[: int(torch.tensor(self.out_shape).prod())].view(*self.out_shape)

    def check_inputs(self, inputs):
        """The plan is frozen for one set of input shapes: anything else is an error (Tensor.copy_ would
        silently broadcast a smaller batch into the static buffer)."""
        if self.multi != isinstance(inputs, (list, tuple)):
            raise RuntimeError("this plan was compiled for %s" % ("a list of pathway tensors" if self.multi else "a single tensor"))
        ins = list(inputs) if self.multi else [inputs]
        if len(ins) != len(self.static_in):
            raise RuntimeError("expected %d input tensors, got %d" % (len(self.static_in), len(ins)))
        for i, (s, t) in enumerate(zip(self.static_in, ins)):
            if not torch.is_tensor(t) or tuple(t.shape) != tuple(s.shape):
                raise RuntimeError("input shape %s differs from the compiled shape %s (compile a plan per shape)" % (
                    tuple(t.shape) if torch.is_tensor(t) else type(t).__name__, tuple(s.shape)))
            if i in self.mask_slots:
                if t.dtype != torch.bool:
                    raise RuntimeError("input %d is a mask: expected a bool tensor, got %s" % (i, t.dtype))
            elif not (t.is_floating_point() or t.dtype == torch.uint8):
                raise RuntimeError("unsupported input dtype %s" % t.dtype)
        return ins

    def side_outputs(self):
        """[(module, device tensor, shape)] of the per-module results of the last replay (attention weights)."""
        outs = [(ref(), b.tensor[:int(torch.tensor(shape).prod())], shape) for ref, b, shape in self.plan.side_outputs]
        return [o for o in outs if o[0] is not None]

    def __call__(self, inputs):
        ins = self.check_inputs(inputs)
        dev = self.plan.device
        with torch.cuda.device(dev):
            for s, t in zip(self.static_in, ins):
                if t.data_ptr() != s.data_ptr():
                    s.copy_(t, non_blocking=True)     # H2D or D2D staging into the plan's static input
            if self.use_graph:
                if self.graph is None:
                    self._capture()
                self.graph.replay()
            else:
                self.plan.run(torch.cuda.current_stream(dev).cuda_stream)
        return self.output_view()


def _raw_inputs(model, ins):
    """Indices of inputs that are not clips / tokens: the trailing [K, 5] box tensor of the detection modules
    (DetectionBBoxNetwork.forward(x, bboxes), ResNetRoIHead.forward(x, bboxes))."""
    if type(model).__name__ in ("DetectionBBoxNetwork", "ResNetRoIHead"):
        b = ins[-1]
        if len(ins) < 2 or b.dim() != 2 or b.shape[1] != 5 or b.shape[0] < 1:
            raise RuntimeError("bboxes must be a [K, 5] tensor (batch index, x1, y1, x2, y2) with K >= 1; "
                               "RoIAlignRotated ([K, 6]) is unsupported")
        return {len(ins) - 1}
    return set()


def _masked_root(extra):
    return bool(extra) and isinstance(extra[0], tuple) and len(extra[0]) >= 2 and extra[0][0] == "masks"


def _mask_slots(ins, extra):
    """Indices of the bool (B, T) masks of a masked module's inputs.  Masked modules call the engine with a flat list
    [x0, (mask0), x1, (mask1), ...] and extra[0] = ("masks", multi, has_mask0, has_mask1, ...)."""
    if not _masked_root(extra):
        return set()
    slots, i = set(), 0
    for has in extra[0][2:]:
        if has:
            slots.add(i + 1)
        i += 2 if has else 1
    if i != len(ins):
        raise RuntimeError("masked inputs: %d tensors for the layout %s" % (len(ins), extra[0]))
    return slots


def _root_input(xs, ins, extra):
    """The (x, mask_ref) pair - or the list of pairs of a MaskedMultiPathWay - a masked root module is lowered on."""
    pairs, i = [], 0
    for has in extra[0][2:]:
        x = xs[i]
        pairs.append((x, xs[i + 1] if has else None))
        i += 2 if has else 1
    return pairs if extra[0][1] else pairs[0]


def _image_root(model, ins):
    """True when the input is one (B, C, H, W) image batch for an image MViT (``patch_embed.patch_model`` a Conv2d,
    create_multiscale_vision_transformers(use_2d_patch=True)); it runs as a clip of one frame.  A 4-D input to any
    other module raises."""
    if not any(torch.is_tensor(t) and t.dim() == 4 for t in ins):
        return False
    pm = getattr(getattr(model, "patch_embed", None), "patch_model", None)
    if type(model).__name__ != "MultiscaleVisionTransformers" or not isinstance(pm, nn.Conv2d) or len(ins) != 1:
        raise RuntimeError("a 4-D (B, C, H, W) input is taken only by an image MViT (patch_embed.patch_model a Conv2d); "
                           "%s expects 5-D (B, C, T, H, W) clips or (B, N, C) tokens" % type(model).__name__)
    return True


def _emit_input(plan, t):
    if t.dim() == 4:              # an image batch (see _image_root): a one-frame clip over the same storage
        x = _emit_input(plan, t.unsqueeze(2))
        x.image = True
        return x
    if t.dim() == 5:
        return plan.emit_input_ncdhw(t, t.shape[1], 4 if t.shape[1] <= 4 else (t.shape[1] + 7) // 8 * 8)
    x = plan.emit_input_tokens(t)
    if t.dim() == 2:
        x.squeeze = True          # a (batch, feature) input: lowerings that keep its rank hand the mark on
    return x


def _emit_output(plan, out, tokens):
    if isinstance(out, TRef):
        if tokens or (out.T == 1 and out.H == 1 and getattr(out, "is_tokens", False)):
            return plan.emit_to_tokens(out, "output.to_tokens", squeeze=getattr(out, "squeeze", False))
        return plan.emit_to_ncdhw(out, "output.to_ncdhw")
    if isinstance(out, list):
        raise NotImplementedError("models returning a list are unsupported")
    return out


def compile_model(model, example_inputs, dtype="f16", use_graph=True, extra=()):
    return CompiledModel(model, example_inputs, dtype, use_graph, extra)


def lower_only(model, example_inputs, dtype="f16", extra=()):
    """Host-side dry run (works without a GPU): build the plan on the CPU and return
    (plan, output_shape).  Nothing can be executed; used by the CPU test-suite to check the
    lowering, shape inference, channel padding, concat fusion and algorithm selection."""
    multi = isinstance(example_inputs, (list, tuple))
    ins = list(example_inputs) if multi else [example_inputs]
    plan = Plan("cpu", {"f16": L.PV_F16, "f32": L.PV_F32}[dtype])
    raw = _raw_inputs(model, ins)
    masks = _mask_slots(ins, extra)
    _image_root(model, ins)
    xs = [plan.raw_input(torch.empty(t.shape, dtype=torch.float32)) if i in raw
          else PL.MaskRef(t.shape[0], t.shape[1], tensor=torch.empty(t.shape, dtype=torch.uint8)) if i in masks
          else _emit_input(plan, torch.empty(t.shape, dtype=torch.float32)) for i, t in enumerate(ins)]
    low = Lowering(plan, extra)
    out = low.lower(model, _root_input(xs, ins, extra) if _masked_root(extra) else (xs if multi else xs[0]), "")
    out = _emit_output(plan, out, tokens=ins[0].dim() not in (4, 5))
    plan.aux = low.aux_out
    return plan, out[1]


# =============================================================================================
# MViT lowering (models/vision_transformers.py:172-182, layers/attention.py)
# =============================================================================================
from . import plan as PL  # noqa: E402


def _check_thw(x, thw, has_cls, name):
    T, H, W = (int(v) for v in thw)
    if x.npos != (1 if has_cls else 0) + T * H * W:
        raise RuntimeError("%s: %d tokens do not match thw_shape %s%s" % (name, x.npos, (T, H, W), " + cls" if has_cls else ""))
    return (T, H, W)


def _folded(weight, bias, fold):
    """A Linear that consumes ``s * x + t`` (an eval BatchNorm1d folded away, ``fold = (s, t)``) as one on x:
    W diag(s), W t + bias."""
    if fold is None:
        return weight, bias
    s, t = fold
    w = weight.detach().float().cpu()
    b = w @ t + (bias.detach().float().cpu() if bias is not None else 0.0)
    return w * s[None, :], b


def _attention_pool(attn, branch):
    """(pool, norm, norm_before_pool) of the _AttentionPool wrapper ``_attention_pool_<branch>`` - what forward calls
    (after fuse_bn() attn.norm_<branch> is an Identity while the wrapper still holds the BatchNorm3d)."""
    ap = getattr(attn, "_attention_pool_" + branch)
    pool = ap.pool if ap.has_pool else None
    norm = ap.norm if ap.has_norm else None
    return pool, norm, bool(ap.has_norm and ap.norm_before_pool)


def _lower_mvit_attention(low, attn, xn, thw, name, residual=None, fold=None):
    """MultiScaleAttention.forward (layers/attention.py:501-544) on normalised tokens ``xn`` (or on x with the block's
    BatchNorm1d ``fold`` = (s, t) folded into the q/k/v projections): returns (proj(attention) [+ residual fused into
    the GEMM epilogue], pooled q thw)."""
    p = low.p
    if getattr(attn, "pool_first", False):
        return _lower_mvit_attention_pool_first(low, attn, xn, thw, name, residual)
    has_cls = attn.has_cls_embed
    heads, dim_att = attn.num_heads, attn.dim_out
    thw = _check_thw(xn, thw, has_cls, name)
    # q/k/v projections as ONE GEMM over concatenated weights; q, k, v are channel slices of its output
    if attn.separate_qkv:
        w = torch.cat([attn.q.weight, attn.k.weight, attn.v.weight], 0)
        b = None if attn.q.bias is None else torch.cat([attn.q.bias, attn.k.bias, attn.v.bias], 0)
    else:
        w, b = attn.qkv.weight, attn.qkv.bias
    w, b = _folded(w, b, fold)
    qkv = PL.emit_linear(p, xn, w, b, L.ACT_NONE, None, name + ".qkv")
    q, k, v = (PL.channel_slice(qkv, i * dim_att, dim_att) for i in range(3))
    thw_q = thw
    pool_q, norm_q, before_q = _attention_pool(attn, "q")
    if pool_q is not None:
        q, thw_q = PL.emit_token_pool(p, q, thw, pool_q, norm_q, heads, has_cls, name + ".pool_q", before_q)
    pool_k, norm_k, before_k = _attention_pool(attn, "k")
    pool_v, norm_v, before_v = _attention_pool(attn, "v")
    if pool_k is not None and pool_v is not None and PL.pools_fusable(pool_k, pool_v, norm_k, norm_v, before_k, before_v):
        # k | v are adjacent channel slices of the QKV GEMM output: ONE depthwise launch (+ ONE LayerNorm launch) for both
        kv, _ = PL.emit_token_pool(p, PL.channel_slice(qkv, dim_att, 2 * dim_att), thw, (pool_k, pool_v), (norm_k, norm_v),
                                   heads, has_cls, name + ".pool_kv", before_k)
        k, v = PL.channel_slice(kv, 0, dim_att), PL.channel_slice(kv, dim_att, dim_att)
    else:
        if pool_k is not None:
            k, _ = PL.emit_token_pool(p, k, thw, pool_k, norm_k, heads, has_cls, name + ".pool_k", before_k)
        if pool_v is not None:
            v, _ = PL.emit_token_pool(p, v, thw, pool_v, norm_v, heads, has_cls, name + ".pool_v", before_v)
    o = PL.emit_attention(p, q, k, v, heads, attn.scale, attn.residual_pool, name + ".core")
    x = PL.emit_linear(p, o, attn.proj.weight, attn.proj.bias, L.ACT_NONE, residual, name + ".proj")
    return x, thw_q


def _lower_mvit_attention_pool_first(low, attn, xn, thw, name, residual=None):
    """pool_first=True (layers/attention.py:511-517): every branch pools the normalised tokens per head (dim // heads
    channels), then its q / k / v linear runs on the pooled tokens; residual_pool adds the projected pooled q."""
    p = low.p
    has_cls = attn.has_cls_embed
    heads = attn.num_heads
    thw = _check_thw(xn, thw, has_cls, name)
    if xn.C % heads:
        raise RuntimeError("%s: %d channels do not split into %d heads" % (name, xn.C, heads))
    outs, thw_q = {}, thw
    for br in ("q", "k", "v"):
        pool, norm, before = _attention_pool(attn, br)
        src = xn
        if pool is not None:
            src, pthw = PL.emit_token_pool(p, xn, thw, pool, norm, heads, has_cls, name + ".pool_" + br, before)
            if br == "q":
                thw_q = pthw
        lin = getattr(attn, br)
        outs[br] = PL.emit_linear(p, src, lin.weight, lin.bias, L.ACT_NONE, None, name + "." + br)
    o = PL.emit_attention(p, outs["q"], outs["k"], outs["v"], heads, attn.scale, attn.residual_pool, name + ".core")
    x = PL.emit_linear(p, o, attn.proj.weight, attn.proj.bias, L.ACT_NONE, residual, name + ".proj")
    return x, thw_q


def _lower_mlp(low, mlp, xn, name, residual=None, fold=None):
    # layers/attention.py:102-114: fc1 -> act -> fc2 (dropout = identity in eval)
    act = _act_code(mlp.act)
    if act == L.ACT_GELU and getattr(mlp.act, "approximate", "none") != "none":
        raise NotImplementedError("Mlp activation must be the exact (erf) GELU")
    w1, b1 = _folded(mlp.fc1.weight, mlp.fc1.bias, fold)
    h = PL.emit_linear(low.p, xn, w1, b1, act, None, name + ".fc1")
    return PL.emit_linear(low.p, h, mlp.fc2.weight, mlp.fc2.bias, L.ACT_NONE, residual, name + ".fc2")


def _norm_kind(m):
    return type(m).__name__


def _block_norms_are_layernorm(blk):
    return _norm_kind(blk.norm1) == "LayerNorm" and _norm_kind(blk.norm2) == "LayerNorm"


def _lower_block_norm(p, x, norm, name, pool_first=False):
    """(x_norm, fold) for a block norm as forward calls it (layers/attention.py:738-742, 748-752): a LayerNorm launch;
    an eval BatchNorm1d folded into the linears that consume x_norm (fold = (s, t), x_norm = x), or - when the attention
    pools x_norm first (zero padding and max / avg do not commute with the affine) - materialised by one launch over
    every row, cls included; an Identity (after fuse_bn()) is x itself."""
    kind = _norm_kind(norm)
    if kind == "LayerNorm":
        return PL.emit_layernorm(p, x, norm, name), None
    if kind == "BatchNorm1d":
        s, t = PL.bn_affine(norm)
        if s.numel() != x.C:
            raise RuntimeError("%s: BatchNorm1d has %d channels, the tokens %d" % (name, s.numel(), x.C))
        if pool_first:
            return PL.emit_channel_affine(p, x, s, t, name), None
        return x, (s, t)
    if kind == "Identity":
        return x, None
    raise NotImplementedError("%s: block norm %s unsupported" % (name, kind))


def _lower_mvit_block(low, blk, x, thw, name, xn=None, next_ln=None, want_sum=True):
    """MultiScaleBlock.forward (layers/attention.py:729-757); DropPath is the identity in eval.
    Returns (x, thw', xn_next).  f16 engine with ``plan.trunk32`` (LayerNorm blocks only): the residual stream x is
    fp32 - the branch outputs (attention proj, fc2) stay f16 and each residual add is fused with the LayerNorm that
    follows it (norm2; ``next_ln`` = the next block's norm1 / the model's norm_embed, whose f16 output comes back as
    xn_next; ``xn`` = this block's already normalised input handed over by the previous block).  BatchNorm1d / Identity
    block norms dispatch on the modules themselves (see _lower_block_norm)."""
    p = low.p
    attn = blk.attn
    has_cls = attn.has_cls_embed
    thw = _check_thw(x, thw, has_cls, name)
    trunk32 = p.trunk32
    assert not trunk32 or _block_norms_are_layernorm(blk)
    fold1 = None
    if xn is None:
        xn, fold1 = _lower_block_norm(p, x, blk.norm1, name + ".norm1", pool_first=getattr(attn, "pool_first", False))
    widen = blk.dim != blk.dim_out
    if blk.dim_mul_in_att and widen:
        w, b = _folded(blk.proj.weight, blk.proj.bias, fold1)
        x = PL.emit_linear(p, xn, w, b, L.ACT_NONE, None, name + ".proj")
    x_res = x
    if getattr(blk, "pool_skip", None) is not None:
        x_res, _ = PL.emit_token_pool(p, x, thw, blk.pool_skip, None, 1, has_cls, name + ".pool_skip")
    if trunk32:
        br, thw_q = _lower_mvit_attention(low, attn, xn, thw, name + ".attn", residual=None)
        x, xn2 = PL.emit_add_layernorm(p, x_res, br, blk.norm2, name + ".norm2")
        fold2 = None
    else:
        x, thw_q = _lower_mvit_attention(low, attn, xn, thw, name + ".attn", residual=x_res, fold=fold1)
        xn2, fold2 = _lower_block_norm(p, x, blk.norm2, name + ".norm2")
    if (not blk.dim_mul_in_att) and widen:
        w, b = _folded(blk.proj.weight, blk.proj.bias, fold2)
        x = PL.emit_linear(p, xn2, w, b, L.ACT_NONE, None, name + ".proj")
    if trunk32:
        br2 = _lower_mlp(low, blk.mlp, xn2, name + ".mlp", residual=None)
        x, xn_next = PL.emit_add_layernorm(p, x, br2, next_ln, name + ".add", want_sum=want_sum or next_ln is None)
        return x, thw_q, xn_next
    x = _lower_mlp(low, blk.mlp, xn2, name + ".mlp", residual=x, fold=fold2)
    return x, thw_q, None


def _pos_table(enc):
    """Rows of the additive table of SpatioTemporalClsPositionalEncoding.forward
    (layers/positional_encoding.py:112-136); row 0 also carries the cls token itself."""
    has_cls = bool(enc.cls_embed_on)
    with torch.no_grad():
        if enc.sep_pos_embed:
            pos = enc.pos_embed_spatial.detach().float().cpu().repeat(1, enc.num_temporal_patch, 1) + \
                torch.repeat_interleave(enc.pos_embed_temporal.detach().float().cpu(), enc.num_spatial_patch, dim=1)
            if has_cls:
                pos = torch.cat([enc.pos_embed_class.detach().float().cpu(), pos], 1)
        else:
            pos = enc.pos_embed.detach().float().cpu().clone()
        pos = pos[0].clone()
        if has_cls:
            pos[0] += enc.cls_token.detach().float().cpu()[0, 0]
    return pos, has_cls


def _lower_vit_head(low, head, x, name="head"):
    """VisionTransformerBasicHead.forward (models/head.py:521-535) on (already normalised) tokens."""
    p = low.p
    mode = head.sequence_pool.mode if head.sequence_pool is not None else None
    if mode == "cls":
        if x.npos > 1:
            x = TRef(x.buf, x.N, 1, 1, 1, x.C, Cp=x.C, ch_off=x.ch_off, row_stride=x.npos * x.row_stride)
    elif mode == "mean":
        x = p.emit_pool(x, L.POOL_AVG, (1, 1, x.W), (1, 1, x.W), (0, 0, 0), name + ".sequence_pool")
    else:
        raise NotImplementedError("sequence_pool=None MViT heads are unsupported")
    x = PL.emit_linear(p, x, head.proj.weight, head.proj.bias, L.ACT_NONE, None, name + ".proj")
    act = head.activation
    softmax = False
    if act is not None:
        if type(act).__name__ == "Softmax":
            softmax = True
        elif type(act).__name__ == "Sigmoid":
            x = p.emit_act(x, L.ACT_SIGMOID, name + ".activation")
        else:
            raise NotImplementedError("head activation unsupported")
    return p.emit_head_reduce(x, softmax, name + ".output")


def _lower_mvit(self, m, x, name):
    p = self.p
    pe = m.patch_embed
    enc = m.cls_positional_encoding
    T, H, W = enc.patch_embed_shape()
    pos, has_cls = _pos_table(enc)
    if type(pe).__name__ == "Identity":
        # enable_patch_embed=False: the input already is the (B, T*H*W, C) patch-token tensor, C the width of the
        # positional table (cls_token is a 0-d placeholder when cls_embed_on=False)
        if x.T != 1 or x.H != 1:
            raise RuntimeError("an MViT without a patch embedding takes (B, T*H*W, C) tokens")
        if x.npos != T * H * W or x.C != pos.shape[1]:
            raise RuntimeError("expected (B, %d, %d) tokens for the %s patch grid, got (B, %d, %d)" % (
                T * H * W, pos.shape[1], (T, H, W), x.npos, x.C))
        pm = None
    elif type(pe).__name__ != "PatchEmbed":
        raise NotImplementedError("MViT patch embedding %s unsupported" % type(pe).__name__)
    else:
        pm = pe.patch_model
    if pm is None:
        pass
    elif isinstance(pm, nn.Conv2d):
        # image MViT (vision_transformers.py use_2d_patch=True): the Conv2d runs as a (1, kh, kw) Conv3d on the
        # one-frame clip, so a 7x7 / stride 4 embed takes the window-mode tensor-core stem like the video models'
        if not getattr(x, "image", False):
            raise RuntimeError("an image MViT (Conv2d patch embedding) takes (B, C, H, W) images")
        if isinstance(pm.padding, str) or pm.padding_mode != "zeros":
            raise NotImplementedError("patch_embed.patch_model: string padding / padding_mode unsupported")
        x = self.p.emit_conv(x, pm.weight.unsqueeze(2), pm.bias, None, (1,) + tuple(pm.stride), (0,) + tuple(pm.padding),
                             (1,) + tuple(pm.dilation), pm.groups, L.ACT_NONE, None, "patch_embed.patch_model")
    else:
        x = self.conv(x, pm, None, None, None, "patch_embed.patch_model")
    if pm is not None and (x.T, x.H, x.W) != (T, H, W):
        raise RuntimeError("input clip gives a %s patch grid but the model was built for %s" % ((x.T, x.H, x.W), (T, H, W)))
    ne = m.norm_embed
    ne_is_ln = type(ne).__name__ == "LayerNorm"
    if p.trunk32 and not (ne_is_ln and all(_block_norms_are_layernorm(b) for b in m.blocks)):
        # the head's GEMM needs f16 tokens: without a final LayerNorm keep the f16 stream; the fp32 trunk also fuses
        # every residual add with a LayerNorm, so BatchNorm / Identity block norms keep it too
        p.trunk32 = False
    x = PL.emit_pos_cls(p, x, pos, has_cls, "cls_positional_encoding", out_dt=L.PV_F32 if p.trunk32 else None)
    thw = (T, H, W)
    xn = None
    nb = len(m.blocks)
    for i, blk in enumerate(m.blocks):
        last = i + 1 == nb
        nxt = (ne if last else m.blocks[i + 1].norm1) if p.trunk32 else None
        x, thw, xn = _lower_mvit_block(self, blk, x, thw, "blocks.%d" % i, xn=xn, next_ln=nxt, want_sum=not last)
    head = m.head
    if type(head).__name__ == "Identity":
        # head=None: the (B, N, C) tokens after norm_embed
        if p.trunk32:
            x = xn             # norm_embed was fused into the last block's residual add
        elif ne_is_ln:
            x = PL.emit_layernorm(p, x, ne, "norm_embed")
        elif type(ne).__name__ != "Identity":
            raise NotImplementedError("MViT norm_embed %s unsupported" % type(ne).__name__)
        return _tok_out(x)
    if type(head).__name__ != "VisionTransformerBasicHead":
        raise NotImplementedError("MViT head %s unsupported" % type(head).__name__)
    mode = head.sequence_pool.mode if head.sequence_pool is not None else None
    if p.trunk32:
        x = xn                 # norm_embed was fused into the last block's residual add
    elif ne_is_ln:
        if mode == "cls":      # only the cls row reaches the head: normalise just those B rows
            x = PL.emit_layernorm(p, x, ne, "norm_embed", rows_stride=x.npos * x.row_stride, rows=x.N)
        else:
            x = PL.emit_layernorm(p, x, ne, "norm_embed")
    return _lower_vit_head(self, head, x, "head")


# ---- layer-level entry points: the MViT building blocks as stand-alone modules (token tensors in / out) ----
def _tok_out(x, squeeze=False):
    x.is_tokens = True
    x.squeeze = squeeze
    return x


def _lower_block_module(self, m, x, name):
    if len(self.extra) != 1:
        raise RuntimeError("MultiScaleBlock.forward(x, thw_shape): thw_shape is required")
    if not _block_norms_are_layernorm(m):
        self.p.trunk32 = False      # the fp32 trunk fuses the residual adds with LayerNorms (see _lower_mvit)
    y, thw, _ = _lower_mvit_block(self, m, x, self.extra[0], name or "block")
    self.aux_out = list(thw)
    return _tok_out(y)


def _lower_attention_module(self, m, x, name):
    if len(self.extra) != 1:
        raise RuntimeError("MultiScaleAttention.forward(x, thw_shape): thw_shape is required")
    y, thw = _lower_mvit_attention(self, m, x, self.extra[0], name or "attn")
    self.aux_out = list(thw)
    return _tok_out(y)


def _lower_mlp_module(self, m, x, name):
    return _tok_out(_lower_mlp(self, m, x, name or "mlp"), squeeze=True)


def _lower_posenc_module(self, m, x, name):
    pos, has_cls = _pos_table(m)
    T, H, W = m.patch_embed_shape()
    if x.npos != T * H * W:
        raise RuntimeError("expected %d patch tokens, got %d" % (T * H * W, x.npos))
    return _tok_out(PL.emit_pos_cls(self.p, x, pos, has_cls, name or "cls_positional_encoding"))


def _lower_patch_embed_module(self, m, x, name):
    # stem.py:289-292: conv then flatten(2).transpose(1, 2) - the NDHWC conv output already is (B, THW, C)
    y = self.conv(x, m.patch_model, None, None, None, (name + "." if name else "") + "patch_model")
    t = TRef(y.buf, y.N, 1, 1, y.npos, y.C, Cp=y.Cp, ch_off=y.ch_off, row_stride=y.row_stride)
    return _tok_out(t)


def _lower_vit_head_module(self, m, x, name):
    return _lower_vit_head(self, m, x, name or "head")


def _lower_sequence_pool_module(self, m, x, name):
    if m.mode == "cls":
        t = TRef(x.buf, x.N, 1, 1, 1, x.C, Cp=x.C, ch_off=x.ch_off, row_stride=x.npos * x.row_stride)
    else:
        t = self.p.emit_pool(x, L.POOL_AVG, (1, 1, x.W), (1, 1, x.W), (0, 0, 0), name or "sequence_pool")
    return _tok_out(t, squeeze=True)


Lowering.lower_MultiScaleBlock = _lower_block_module
Lowering.lower_MultiScaleAttention = _lower_attention_module
Lowering.lower_Mlp = _lower_mlp_module
Lowering.lower_SpatioTemporalClsPositionalEncoding = _lower_posenc_module
Lowering.lower_PatchEmbed = _lower_patch_embed_module
Lowering.lower_VisionTransformerBasicHead = _lower_vit_head_module
Lowering.lower_SequencePool = _lower_sequence_pool_module
Lowering.lower_MultiscaleVisionTransformers = _lower_mvit


# =============================================================================================
# Masked multistream lowering (models/masked_multistream.py, layers/fusion.py, layers/positional_encoding.py:11-44).
# A masked handler takes (x, mask) and returns (y, mask): the attention modules hand the mask with its first column
# forced valid (:137-141, :309-313) to the modules after them, as the reference's in-place write does.  Token tensors
# are TRef(B, 1, 1, T, C); ``squeeze`` marks a (batch, feature) tensor, ``retargetable`` a result whose producer
# resolves its row stride at run time, so that ConcatFusion can move it into a channel slice.
# =============================================================================================
_MASK_MODULES = ("MaskedTemporalPooling", "LearnMaskedDefault", "TransposeMultiheadAttention", "LSTM",
                 "TransposeTransformerEncoder")
_MASKED_HEAD_DIMS = (32, 64, 96, 128)
_MPOOL = {"max": L.MPOOL_MAX, "avg": L.MPOOL_AVG, "sum": L.MPOOL_SUM}


def _is_mask_module(m):
    n = type(m).__name__
    return n in _MASK_MODULES and (n != "LSTM" or hasattr(m, "lstm"))       # a plain nn.LSTM takes no mask


def _mark(y, x=None, squeeze=None, retargetable=False):
    y.squeeze = getattr(x, "squeeze", False) if squeeze is None else squeeze
    y.retargetable = retargetable
    return y


def _token_input(x, name, what):
    if not isinstance(x, TRef) or x.T != 1 or x.H != 1 or x.lazy_src is not None:
        raise NotImplementedError("%s: %s runs on (batch, seq_len, feature) token tensors only" % (name, what))


def _check_mask(x, mask, name):
    if mask is not None and (mask.B != x.N or mask.T != x.npos):
        raise RuntimeError("%s: mask of shape %s for x with (batch, seq_len) = %s" % (name, (mask.B, mask.T),
                                                                                      (x.N, x.npos)))


def _seq3(x, name):
    if getattr(x, "squeeze", False):
        raise RuntimeError("%s: requires x shape (batch_size x seq_len x feature_dim)" % name)


def _mha_check(a, name):
    if not getattr(a, "_qkv_same_embed_dim", True) or a.bias_k is not None or a.add_zero_attn or \
            getattr(a, "batch_first", False):
        raise NotImplementedError("%s: MultiheadAttention variant unsupported (kdim / vdim, bias_kv, add_zero_attn, "
                                  "batch_first)" % name)
    D = a.embed_dim // a.num_heads
    if D not in _MASKED_HEAD_DIMS:
        raise NotImplementedError("%s: head dim %d (embed_dim %d / num_heads %d) has no masked attention kernel "
                                  "(supported: %s)" % (name, D, a.embed_dim, a.num_heads, _MASKED_HEAD_DIMS))
    return D


def _mha(low, a, x, mask, name, weights):
    """nn.MultiheadAttention(x, x, x, key_padding_mask=~mask): the in-projection as one GEMM, the key-masked attention,
    the out-projection.  Returns (in-projection-free attention output o, weights Buf or None)."""
    p = low.p
    D = _mha_check(a, name)
    if x.C != a.embed_dim:
        raise RuntimeError("%s: embed_dim %d, input has %d features" % (name, a.embed_dim, x.C))
    qkv = PL.emit_linear(p, x, a.in_proj_weight, a.in_proj_bias, L.ACT_NONE, None, name + ".in_proj")
    F = a.embed_dim
    q, k, v = (PL.channel_slice(qkv, i * F, F) for i in range(3))
    return PL.emit_attention_masked(p, q, k, v, a.num_heads, D ** -0.5, mask, name + ".attention", weights=weights)


def _masked_pool(low, m, x, mask, name):
    _seq3(x, name)
    _check_mask(x, mask, name)
    return _mark(PL.emit_masked_pool(low.p, x, mask, _MPOOL[m._method], name), squeeze=True, retargetable=True), mask


def _learned_default(low, m, x, mask, name):
    if mask is not None:
        if mask.B != x.N:
            raise RuntimeError("%s: mask batch %d, x batch %d" % (name, mask.B, x.N))
    return _mark(PL.emit_masked_default(low.p, x, mask, m._learned_defaults, name), x, retargetable=True), mask


def _transpose_mha(low, m, x, mask, name):
    _seq3(x, name)
    _check_mask(x, mask, name)
    a = m._attention
    _mha_check(a, name + "._attention")
    if mask is not None:
        mask = PL.emit_mask_force_first(low.p, mask, name + ".mask")
    o, w = _mha(low, a, x, mask, name + "._attention", weights=True)
    y = PL.emit_linear(low.p, o, a.out_proj.weight, a.out_proj.bias, L.ACT_NONE, None, name + "._attention.out_proj")
    # a weak reference: the module holds its compiled plans, and a plan that held the module back would put the plan's
    # CUDA graph in a reference cycle, freed by the garbage collector at an arbitrary moment - possibly inside another
    # plan's graph capture, which the graph's destruction would invalidate
    low.p.side_outputs.append((weakref.ref(m), w, (x.N, x.npos, x.npos)))
    return _mark(y, x, retargetable=True), mask


def _encoder(low, m, x, mask, name):
    """nn.TransformerEncoder of post-norm layers (torch's slow path, which the reference's batch_first=False layers
    take): x = norm1(x + out_proj(attn(x))); x = norm2(x + linear2(relu(linear1(x)))); the result is position 0."""
    _seq3(x, name)
    _check_mask(x, mask, name)
    p = low.p
    enc = m.encoder
    layers = list(enc.layers)
    for i, lyr in enumerate(layers):
        lname = "%s.encoder.layers.%d" % (name, i)
        if getattr(lyr, "norm_first", False):
            raise NotImplementedError("%s: norm_first (pre-norm) layers are unsupported" % lname)
        act = lyr.activation
        if not (act is torch.nn.functional.relu or type(act).__name__ == "ReLU"):
            raise NotImplementedError("%s: activation %s unsupported (ReLU only)" % (lname, getattr(act, "__name__", act)))
        _mha_check(lyr.self_attn, lname + ".self_attn")
    if mask is not None:
        mask = PL.emit_mask_force_first(p, mask, name + ".mask")
    for i, lyr in enumerate(layers):
        lname = "%s.encoder.layers.%d" % (name, i)
        a = lyr.self_attn
        o, _ = _mha(low, a, x, mask, lname + ".self_attn", weights=False)
        h = PL.emit_linear(p, o, a.out_proj.weight, a.out_proj.bias, L.ACT_NONE, x, lname + ".self_attn.out_proj")
        x = PL.emit_layernorm(p, h, lyr.norm1, lname + ".norm1")
        f = PL.emit_linear(p, x, lyr.linear1.weight, lyr.linear1.bias, L.ACT_RELU, None, lname + ".linear1")
        h = PL.emit_linear(p, f, lyr.linear2.weight, lyr.linear2.bias, L.ACT_NONE, x, lname + ".linear2")
        x = PL.emit_layernorm(p, h, lyr.norm2, lname + ".norm2")
    if enc.norm is not None:
        x = PL.emit_layernorm(p, x, enc.norm, name + ".encoder.norm")
    first = TRef(x.buf, x.N, 1, 1, 1, x.C, Cp=x.C, ch_off=x.ch_off, row_stride=x.npos * x.row_stride)   # out[:, 0, :]
    return _mark(first, squeeze=True), mask


_LSTM_MAX_HIDDEN = 512       # csrc/pv_lstm.cu: one thread per hidden unit


def _lstm(low, m, x, mask, name):
    """LSTM.forward (:227-256): one token GEMM for the input projection of both directions ([W_ih_fwd; W_ih_rev], bias
    b_ih + b_hh), then the recurrence of every step and direction in one launch; the output is h_n, [B, ndir * H]."""
    _seq3(x, name)
    _check_mask(x, mask, name)
    r = m.lstm
    H = r.hidden_size
    if r.num_layers != 1 or not r.batch_first or getattr(r, "proj_size", 0) or r.mode != "LSTM":
        raise NotImplementedError("%s: only the single-layer batch_first LSTM of the reference is supported" % name)
    if H > _LSTM_MAX_HIDDEN:
        raise NotImplementedError("%s: LSTM hidden_dim=%d has no recurrence kernel (at most %d)" % (
            name, H, _LSTM_MAX_HIDDEN))
    if r.input_size != x.C:
        raise RuntimeError("%s: LSTM dim_in %d, input has %d features" % (name, r.input_size, x.C))
    p = low.p
    sfx = ["", "_reverse"][:2 if r.bidirectional else 1]
    nd = len(sfx)

    def par(n, s_):
        t = getattr(r, n + "_l0" + s_, None)
        return None if t is None else t.detach().float().cpu()
    w_ih = torch.cat([par("weight_ih", s_) for s_ in sfx], 0)
    bias = None
    if r.bias:
        bias = torch.cat([par("bias_ih", s_) + par("bias_hh", s_) for s_ in sfx], 0)
    g = PL.emit_linear(p, x, w_ih, bias, L.ACT_NONE, None, name + ".lstm.input_proj")
    w_hh = torch.stack([par("weight_hh", s_).t().contiguous() for s_ in sfx], 0)                # [dir][H][4H]
    w_hh_t = p.const(w_hh)
    y = PL._tok(p, x.N, 1, nd * H)
    lib = p.lib
    B, T = x.N, x.npos

    def fn(stream):
        L.check(lib.pv_lstm_recurrence(g.ptr(), g.dt, g.row_stride, w_hh_t.data_ptr(), PL._mask_ptr(mask), B, T, H, nd,
                                       y.ptr(), y.row_stride, stream), "pv_lstm_recurrence(%s)" % name)
    p.add(name + ".lstm.recurrence", fn, "other", 2.0 * nd * B * T * 4 * H * H, nd * 4 * H * H * 4 * T,
          reads=(g,) + PL._mask_io(mask), writes=(y,),
          spec={"kind": "lstm", "g": g, "mask": mask, "y": y, "w_hh_t": w_hh, "hidden": H, "dirs": nd})
    return _mark(y, squeeze=True, retargetable=True), mask


_MASKED_LOWERINGS = {"MaskedTemporalPooling": _masked_pool, "LearnMaskedDefault": _learned_default,
                     "TransposeMultiheadAttention": _transpose_mha, "TransposeTransformerEncoder": _encoder,
                     "LSTM": _lstm}


def _lower_masked(low, m, x, mask, name):
    n = type(m).__name__
    if n == "MaskedSequential":
        return _masked_sequential(low, m, x, mask, name)
    if not _is_mask_module(m):
        raise NotImplementedError("%s: %s takes no mask (a stream must be a MaskedSequential or a mask module)" % (name, n))
    return _MASKED_LOWERINGS[n](low, m, x, mask, name)


def _masked_sequential(low, m, x, mask, name):
    # models/masked_multistream.py:338-344: mask modules get (input, mask), the others the input alone
    for i, child in enumerate(m):
        cname = "%s.%d" % (name, i) if name else str(i)
        if _is_mask_module(child):
            x, mask = _lower_masked(low, child, x, mask, cname)
        else:
            x = low.lower(child, x, cname)
    return x, mask


def _root_handler(fn):
    def lower(self, m, x, name):
        if type(m).__name__ != "MaskedSequential" and not _is_mask_module(m):
            raise NotImplementedError("no B200 lowering for module %s (%s)" % (type(m).__name__, name))
        if not isinstance(x, tuple) or len(x) != 2:
            raise RuntimeError("%s.forward takes (x, mask)" % type(m).__name__)
        return fn(self, m, x[0], x[1], name or ("" if type(m).__name__ == "MaskedSequential" else type(m).__name__))[0]
    return lower


def _lower_multipathway(self, m, x, name):
    # models/masked_multistream.py:372-384; every stream runs on its own lane until the fusion
    if m.multipathway_fusion is None:
        raise RuntimeError("MaskedMultiPathWay needs a multipathway_fusion to reduce its streams")
    outs = []
    for i, (blk, (xi, mi)) in enumerate(zip(m.multipathway_blocks, x)):
        self.p.lane = i
        outs.append(_lower_masked(self, blk, xi, mi, "%s.multipathway_blocks.%d" % (name, i) if name
                                  else "multipathway_blocks.%d" % i)[0])
    self.p.lane = 0
    return self.lower(m.multipathway_fusion, outs, (name + "." if name else "") + "multipathway_fusion")


def reduce_fusion_op(reduce_fn):
    """Classify ReduceFusion's opaque reduce_fn on a fixed CPU probe: max gives 3, sum 5, prod 6."""
    try:
        with torch.no_grad():
            r = reduce_fn(torch.tensor([[2.0], [3.0]]))
        v = float(r.reshape(-1)[0]) if torch.is_tensor(r) and r.numel() == 1 else None
    except Exception as e:       # noqa: BLE001 - any failure means the function is not one of the three
        raise NotImplementedError("ReduceFusion: reduce_fn is not max / sum / prod over dim 0 (%s)" % e) from None
    op = {3.0: L.REDUCE_MAX, 5.0: L.REDUCE_SUM, 6.0: L.REDUCE_PROD}.get(v)
    if op is None:
        raise NotImplementedError("ReduceFusion: reduce_fn gives %r on the probe [[2], [3]]; only max (3), sum (5) and "
                                  "prod (6) over dim 0 have a kernel" % (v,))
    return op


def _fusion_parts(x, name):
    if not isinstance(x, (list, tuple)) or not x:
        raise RuntimeError("%s: a fusion layer takes a non-empty list of tensors" % name)
    for t in x:
        _token_input(t, name, "fusion")
    return list(x)


def _concat_last(low, parts, name):
    p0 = parts[0]
    moved = []
    for i, t in enumerate(parts):
        if (t.N, t.npos) != (p0.N, p0.npos) or getattr(t, "squeeze", False) != getattr(p0, "squeeze", False):
            raise RuntimeError("%s: inputs of different shapes" % name)
        PL._dense8(t, name)
        if not getattr(t, "retargetable", False) or any(t is u for u in moved):
            c = PL._tok(low.p, t.N, t.npos, t.C)
            PL.emit_copy_tokens(low.p, t, c, 0, "%s.copy%d" % (name, i))
            t = _mark(c, t, retargetable=True)
        moved.append(t)
    return _mark(low.p.concat_channels(moved), p0) if len(moved) > 1 else moved[0]


def _lower_concat_fusion(self, m, x, name):
    # layers/fusion.py:46-74, torch.cat(input_list, dim=-1): the producers write channel slices of one buffer
    return _concat_last(self, _fusion_parts(x, name or "fusion"), name or "fusion")


def _lower_temporal_concat_fusion(self, m, x, name):
    # layers/fusion.py:77-101, torch.cat(input_list, dim=1): (batch, feature) inputs concatenate their features
    name = name or "fusion"
    parts = _fusion_parts(x, name)
    if all(getattr(t, "squeeze", False) for t in parts):
        return _concat_last(self, parts, name)
    p0 = parts[0]
    for t in parts:
        if t.N != p0.N or t.C != p0.C or getattr(t, "squeeze", False):
            raise RuntimeError("%s: inputs of different batch / feature sizes" % name)
        PL._dense8(t, name)
    y = PL._tok(self.p, p0.N, sum(t.npos for t in parts), p0.C)
    row = 0
    for i, t in enumerate(parts):
        PL.emit_copy_tokens(self.p, t, y, row, "%s.copy%d" % (name, i))
        row += t.npos
    return _mark(y, retargetable=True)


def _lower_reduce_fusion(self, m, x, name):
    # layers/fusion.py:104-141, reduce_fn(torch.stack(input_list)) for max / sum / prod over dim 0
    name = name or "fusion"
    op = reduce_fusion_op(m.reduce_fn)
    parts = _fusion_parts(x, name)
    for t in parts:
        if getattr(t, "squeeze", False) != getattr(parts[0], "squeeze", False):
            raise RuntimeError("%s: inputs of different shapes" % name)
    return _mark(PL.emit_reduce_fusion(self.p, parts, op, name), parts[0], retargetable=True)


def _lower_layernorm(self, m, x, name):
    name = name or "layernorm"
    _token_input(x, name, "LayerNorm")
    if tuple(m.normalized_shape) != (x.C,):
        raise RuntimeError("%s: normalized_shape %s, input has %d features" % (name, tuple(m.normalized_shape), x.C))
    if m.weight is None or m.bias is None:
        raise NotImplementedError("%s: LayerNorm without an elementwise affine weight and bias is unsupported" % name)
    PL._dense8(x, name)
    return _mark(PL.emit_layernorm(self.p, x, m, name), x, retargetable=True)


def _lower_linear(self, m, x, name):
    name = name or "linear"
    _token_input(x, name, "Linear")
    if m.in_features != x.C:
        raise RuntimeError("%s: in_features %d, input has %d features" % (name, m.in_features, x.C))
    return _mark(PL.emit_linear(self.p, x, m.weight, m.bias, L.ACT_NONE, None, name), x, retargetable=True)


def _lower_positional_encoding(self, m, x, name):
    name = name or "positional_encoding"
    _token_input(x, name, "PositionalEncoding")
    _seq3(x, name)
    if m.pe.size(1) < x.npos:
        raise RuntimeError("Cannot apply position encoding of size %s when input has %d positions" % (
            tuple(m.pe.size()), x.npos))
    if m.pe.size(2) != x.C:
        raise RuntimeError("%s: embed_dim %d, input has %d features" % (name, m.pe.size(2), x.C))
    PL._dense8(x, name)
    return _mark(PL.emit_pos_cls(self.p, x, m.pe[0, :x.npos].detach().float().cpu(), False, name), x)


for _n, _fn in _MASKED_LOWERINGS.items():
    setattr(Lowering, "lower_" + _n, _root_handler(_fn))
Lowering.lower_MaskedSequential = _root_handler(_masked_sequential)
Lowering.lower_MaskedMultiPathWay = _lower_multipathway
Lowering.lower_ConcatFusion = _lower_concat_fusion
Lowering.lower_TemporalConcatFusion = _lower_temporal_concat_fusion
Lowering.lower_ReduceFusion = _lower_reduce_fusion
Lowering.lower_LayerNorm = _lower_layernorm
Lowering.lower_Linear = _lower_linear
Lowering.lower_PositionalEncoding = _lower_positional_encoding


# =============================================================================================
# Mobile efficient blocks (layers/accelerator/mobile_cpu/, models/accelerator/mobile_cpu/): this package's trees and
# the reference's original-form trees.  Their class names collide with others (SqueezeExcitation, ReLU, Swish,
# Identity), so these handlers also check attributes.  The reference's deployable form (convert() applied: Conv2d
# decompositions, _Reshape, _SkipConnectMul, fused ConvReLU) is refused with the name of the first module met.
# =============================================================================================
_MOBILE_ACTS = ("ReLU", "Swish", "HardSwish", "Identity")


def _deployable(m, name):
    from ..module import B200Module
    if getattr(m, "convert_flag", False) and not isinstance(m, B200Module):
        raise NotImplementedError("%s: %s is in the reference's deployable (converted) form, which has no B200 lowering; "
                                  "lower the original form" % (name, type(m).__name__))


def _se_block(m, name):
    """The fvcore-style Sequential(Conv3d, ReLU, Conv3d, Sigmoid) of a SqueezeExcitation: ``.block`` (fvcore / X3D) or
    ``.se.block`` (the mobile wrapper)."""
    _deployable(m, name)
    se = getattr(m, "se", None)
    blk = getattr(se, "block", None) if se is not None else getattr(m, "block", None)
    if not isinstance(blk, nn.Sequential) or len(blk) != 4:
        raise NotImplementedError("%s: SqueezeExcitation variant %s unsupported" % (
            name, type(se).__name__ if se is not None else "without a block"))
    return blk


def _mobile_parts(m, name):
    """(conv, bn or None, act wrapper) of a mobile convolution block: kernel = Sequential(conv, [bn], act)."""
    _deployable(m, name)
    k = getattr(m, "kernel", None)
    mods = getattr(k, "_modules", {})
    if not isinstance(k, nn.Sequential) or list(mods) not in (["conv", "act"], ["conv", "bn", "act"]) \
            or type(mods["conv"]) is not nn.Conv3d or type(mods["act"]).__name__ not in _MOBILE_ACTS:
        raise NotImplementedError("%s: %s without its original Sequential(conv, [bn], act) kernel has no B200 lowering"
                                  % (name, type(m).__name__))
    return mods["conv"], mods.get("bn"), mods["act"]


def _mobile_conv(self, x, m, name, residual=None, act=None):
    """A mobile convolution block as one convolution; ``act`` (with ``residual``) replaces its own activation, which
    must then be the identity."""
    conv, bn, own = _mobile_parts(m, name)
    if act is not None and type(own).__name__ != "Identity":
        raise NotImplementedError("%s: activation %s before the block's residual add / activation" % (
            name, type(own).__name__))
    return self.conv(x, conv, bn, own if act is None else act, residual, name)


def _lower_mobile_conv(self, m, x, name):
    return _mobile_conv(self, x, m, name or "conv")


def _lower_x3d_bottleneck(self, m, x, name):
    name = name or "block"
    _deployable(m, name)
    layers = m.layers
    keys = [k for k in layers._modules if k != "se"]
    if keys != ["conv_0", "conv_1", "act_func_1", "conv_2"]:
        raise NotImplementedError("%s: X3dBottleneckBlock layers %s unsupported" % (name, list(layers._modules)))
    shortcut = None
    if m._use_residual:       # the shortcut first, as ResBlock's branch1: the same launch order as models/x3d.py
        shortcut = x if m._res_proj is None else _mobile_conv(self, x, m._res_proj, name + "._res_proj")
    h = _mobile_conv(self, x, layers.conv_0, name + ".layers.conv_0")
    se = layers._modules.get("se")
    if se is None:
        h = _mobile_conv(self, h, layers.conv_1, name + ".layers.conv_1", act=layers.act_func_1)
    else:
        blk = _se_block(se, name + ".layers.se")
        if type(blk[1]).__name__ != "ReLU" or type(blk[3]).__name__ != "Sigmoid":
            raise NotImplementedError("%s.layers.se: SqueezeExcitation variant unsupported" % name)
        conv, bn, own = _mobile_parts(layers.conv_1, name + ".layers.conv_1")
        if type(own).__name__ != "Identity":
            raise NotImplementedError("%s.layers.conv_1: activation %s before the SE" % (name, type(own).__name__))
        h = self.conv(h, conv, bn, None, None, name + ".layers.conv_1", se_sums=True)
        h = self.p.emit_se_scale_act(h, blk[0].weight, blk[0].bias, blk[2].weight, blk[2].bias,
                                     _act_code(layers.act_func_1), name + ".layers.se")
    return _mobile_conv(self, h, layers.conv_2, name + ".layers.conv_2", residual=shortcut, act=m.final_act)


def _lower_efficient_x3d(self, m, x, name):
    pre = name + "." if name else ""
    if self.extra != ("head",):          # ("head",): the head alone, on the s5 feature map (EfficientX3d.forward)
        for s in ("s1", "s2", "s3", "s4", "s5"):
            for cname, blk in getattr(m, s).named_children():
                x = self.lower(blk, x, "%s%s.%s" % (pre, s, cname))
    if not m.enable_head:
        return x
    # head (efficient_x3d.py forward): conv_5 -> avg_pool -> lin_5 -> permute -> projection -> act -> mean over the
    # (1, 1, 1) grid -> view (N, -1); the activation goes into the projection's epilogue
    head = m.head
    if list(head._modules) != ["conv_5", "avg_pool", "lin_5"]:
        raise NotImplementedError("%shead: layers %s unsupported" % (pre, list(head._modules)))
    x = _mobile_conv(self, x, head.conv_5, pre + "head.conv_5")
    x = self.lower(head.avg_pool, x, pre + "head.avg_pool")
    x = _mobile_conv(self, x, head.lin_5, pre + "head.lin_5")
    _deployable(m.projection, pre + "projection")
    proj = getattr(m.projection, "model", None)
    if not isinstance(proj, nn.Linear):
        raise NotImplementedError("%sprojection: %s unsupported" % (pre, type(proj).__name__))
    if type(m.act).__name__ not in _MOBILE_ACTS:
        raise NotImplementedError("%sact: %s unsupported" % (pre, type(m.act).__name__))
    w = proj.weight.reshape(proj.out_features, proj.in_features, 1, 1, 1)
    x = self.p.emit_conv(x, w, proj.bias, None, (1, 1, 1), (0, 0, 0), (1, 1, 1), 1, _act_code(m.act), None,
                         pre + "projection")
    return self.p.emit_head_reduce(x, False, pre + "mean")


def _lower_pool_size1(self, m, x, name):
    _deployable(m, name or "pool")
    return self.pool(x, m.pool, name or "pool")


def _lower_no_op_convert(self, m, x, name):
    return self.lower(m.model, x, (name + "." if name else "") + "model")


def _lower_hardswish(self, m, x, name):
    self.p.materialize_input(x)
    return self.p.emit_act(x, L.ACT_HSWISH, name or "hswish")


for _n in ("Conv3dPwBnAct", "Conv3d3x3x3DwBnAct", "Conv3dTemporalKernel1BnAct", "Conv3d3x1x1BnAct", "Conv3d5x1x1BnAct"):
    setattr(Lowering, "lower_" + _n, _lower_mobile_conv)
def _lower_adaptive_avg_pool3d(self, m, x, name):
    # torch.nn.AdaptiveAvgPool3d, or the mobile wrapper of the same name that holds one as ``.model``
    if isinstance(getattr(m, "model", None), nn.Module):
        return _lower_no_op_convert(self, m, x, name)
    return self.pool(x, m, name)


Lowering.lower_NoOpConvertBlock = _lower_no_op_convert
Lowering.lower_FullyConnected = _lower_no_op_convert
Lowering.lower_AdaptiveAvgPool3d = _lower_adaptive_avg_pool3d
Lowering.lower_X3dBottleneckBlock = _lower_x3d_bottleneck
Lowering.lower_EfficientX3d = _lower_efficient_x3d
Lowering.lower_AdaptiveAvgPool3dOutSize1 = _lower_pool_size1
Lowering.lower_HardSwish = _lower_hardswish
Lowering.lower_Hardswish = _lower_hardswish


# =============================================================================================
# Projector MLPs on (B, C) rows (layers/mlp.py make_multilayer_perceptron, the BYOL predictor of models/byol.py:59-64)
# and the headless ResNet trunk they follow (head.py:371-391 with ``proj = None``).  A row tensor is a TRef of
# N rows with T = H = 1 and W = 1 (a pooled clip) or W = tokens (a (B, C) network input).
# =============================================================================================
def _lower_linear_chain(self, mods, i, x, name):
    """``mods[i]`` (a Linear) with an eval BatchNorm (BatchNorm1d, SyncBatchNorm, NaiveSyncBatchNorm1d) and / or a ReLU
    right after it, as ONE GEMM launch: the BatchNorm folds into the epilogue scale and bias (packing.fold_bn), the ReLU
    is the epilogue activation.  Returns (rows, index of the next module)."""
    lin = mods[i]
    lname = "%s.%d" % (name, i)
    _token_input(x, lname, "Linear")
    if lin.in_features != x.C:
        raise RuntimeError("%s: in_features %d, input has %d features" % (lname, lin.in_features, x.C))
    j = i + 1
    bn = None
    if j < len(mods) and _is_bn(mods[j]):
        bn = mods[j]
        if bn.running_mean is None or bn.running_var is None:
            raise NotImplementedError("%s.%d: BatchNorm without running statistics normalises with batch statistics, "
                                      "which the eval-mode engine does not compute" % (name, j))
        if bn.num_features != lin.out_features:
            raise RuntimeError("%s.%d: BatchNorm has %d features, the Linear %d" % (name, j, bn.num_features,
                                                                                  lin.out_features))
        j += 1
    act = L.ACT_NONE
    if j < len(mods) and type(mods[j]).__name__ == "ReLU":
        act = L.ACT_RELU
        j += 1
    w = lin.weight.reshape(lin.out_features, lin.in_features, 1, 1, 1)
    y = self.p.emit_conv(x, w, lin.bias, bn, (1, 1, 1), (0, 0, 0), (1, 1, 1), 1, act, None, lname)
    y.is_tokens = getattr(x, "is_tokens", False)
    return _mark(y, x, retargetable=True), j


def _lower_headless(self, m, x, name):
    """ResNetBasicHead with its projection removed (``blocks[-1].proj = None``, the trunk of a self-supervised
    checkpoint): [pool] -> [activation] -> [output_pool + view(B, -1)], the pooled features as (B, C) rows."""
    act = getattr(m, "activation", None)
    if act is not None:
        an = type(act).__name__
        if an != "Sigmoid":
            raise NotImplementedError("%s: activation %s of a head without proj unsupported" % (name, an))
        x = self.p.emit_act(x, L.ACT_SIGMOID, name + ".activation")
    if getattr(m, "output_pool", None) is None:
        return x
    if x.npos != 1:
        x = self.p.emit_pool(x, L.POOL_AVG, (x.T, x.H, x.W), (x.T, x.H, x.W), (0, 0, 0), name + ".output_pool")
    return _tok_out(x, squeeze=True)
