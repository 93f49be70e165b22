"""Multiscale Vision Transformers (reference models/vision_transformers.py:185-506)."""
import warnings
from functools import partial

import torch
import torch.nn as nn

from ..layers.attention import MultiScaleBlock
from ..layers.positional_encoding import SpatioTemporalClsPositionalEncoding
from ..layers.utils import round_width
from ..module import B200Module
from .head import create_vit_basic_head
from .stem import create_conv_patch_embed
from .weight_init import init_net_weights


class MultiscaleVisionTransformers(B200Module):
    """patch_embed -> cls/pos encoding -> blocks -> norm -> head (vision_transformers.py:17-182).
    ``forward`` compiles the whole tree into one token-major plan (B, 1+THW, C)."""

    def __init__(self, *, patch_embed, cls_positional_encoding, pos_drop, blocks, norm_embed, head):
        super().__init__()
        assert hasattr(cls_positional_encoding, "patch_embed_shape"), \
            "cls_positional_encoding should have method patch_embed_shape."
        self.patch_embed = patch_embed or nn.Identity()
        self.cls_positional_encoding = cls_positional_encoding
        self.pos_drop = pos_drop or nn.Identity()
        self.blocks = blocks
        self.norm_embed = norm_embed or nn.Identity()
        self.head = head or nn.Identity()
        init_net_weights(self, init_std=0.02, style="vit")

    # ---- BatchNorm folding of the norm="batchnorm" model (vision_transformers.py:85-170) ----
    # These rewrite the tree the way the reference's methods do, so state_dict and repr after fuse_bn() are the
    # reference's.  Like the reference, fuse_bn() does NOT preserve the output: it folds attn.norm_{q,k,v} (the
    # BatchNorm3d that forward applies before the pooling conv, under a GELU) after the q/k/v linears, while the
    # _attention_pool_{q,k,v} wrappers keep the BatchNorm3d and still apply it.  forward runs what the tree holds.
    def _get_bn_w_b(self, bn, repeat=1):
        """(diag(gamma / sqrt(var + eps)), beta - gamma * mean / sqrt(var + eps)), both tiled ``repeat`` times."""
        std = torch.sqrt(bn.running_var + bn.eps)
        w = torch.diag((bn.weight / std).repeat(repeat))
        b = (bn.bias - bn.weight * bn.running_mean / std).repeat(repeat)
        return w, b

    @staticmethod
    def _new_linear(weight, bias):
        out = nn.Linear(weight.shape[1], weight.shape[0], bias=True)
        out.weight.data[:] = weight
        out.bias.data[:] = bias
        return out

    def fuse_norm_before_linear(self, bn, linear):
        """linear(bn(x)) as one Linear."""
        if bn is None:
            return linear
        w, b = self._get_bn_w_b(bn)
        bias = linear.weight @ b
        if linear.bias is not None:
            bias = bias + linear.bias
        return self._new_linear(linear.weight @ w, bias)

    def fuse_norm_after_linear(self, linear, bn):
        """bn(linear(x)) as one Linear, bn's channels tiled over the heads."""
        if bn is None:
            return linear
        width = bn.bias.shape[0]
        assert linear.in_features % width == 0
        w, b = self._get_bn_w_b(bn, repeat=linear.in_features // width)
        bias = w @ linear.bias + b if linear.bias is not None else b
        return self._new_linear(w @ linear.weight, bias)

    def fuse_bn(self):
        assert not self.training
        for blk in self.blocks:
            attn = blk.attn
            if attn.separate_qkv:
                attn.q = self.fuse_norm_before_linear(blk.norm1, attn.q)
                attn.k = self.fuse_norm_before_linear(blk.norm1, attn.k)
                attn.v = self.fuse_norm_before_linear(blk.norm1, attn.v)
            else:
                attn.qkv = self.fuse_norm_before_linear(blk.norm1, attn.qkv)
            blk.norm1 = nn.Identity()
            if attn.separate_qkv:
                attn.q = self.fuse_norm_after_linear(attn.q, attn.norm_q)
                attn.k = self.fuse_norm_after_linear(attn.k, attn.norm_k)
                attn.v = self.fuse_norm_after_linear(attn.v, attn.norm_v)
            else:
                ws, bs = attn.qkv.weight.chunk(3), attn.qkv.bias.chunk(3)
                parts = [self.fuse_norm_after_linear(self._new_linear(w, b), n)
                         for w, b, n in zip(ws, bs, (attn.norm_q, attn.norm_k, attn.norm_v))]
                attn.qkv.weight.data[:] = torch.cat([l.weight.data for l in parts], 0)
                attn.qkv.bias.data[:] = torch.cat([l.bias.data for l in parts], 0)
            attn.norm_q = nn.Identity()
            attn.norm_k = nn.Identity()
            attn.norm_v = nn.Identity()
            blk.mlp.fc1 = self.fuse_norm_before_linear(blk.norm2, blk.mlp.fc1)
            if blk.dim != blk.dim_out:
                blk.proj = self.fuse_norm_before_linear(blk.norm2, blk.proj)
            blk.norm2 = nn.Identity()
        for m in self.modules():            # modules were replaced: drop every plan compiled from the old tree
            m.__dict__.pop("_pv_cache", None)
            m.__dict__.pop("_pv_tensors", None)


def create_multiscale_vision_transformers(*, spatial_size, temporal_size, cls_embed_on=True, sep_pos_embed=True,
                                          depth=16, norm="layernorm", enable_patch_embed=True, input_channels=3,
                                          patch_embed_dim=96, conv_patch_embed_kernel=(3, 7, 7),
                                          conv_patch_embed_stride=(2, 4, 4), conv_patch_embed_padding=(1, 3, 3),
                                          enable_patch_embed_norm=False, use_2d_patch=False, num_heads=1,
                                          mlp_ratio=4.0, qkv_bias=True, dropout_rate_block=0.0,
                                          droppath_rate_block=0.0, pooling_mode="conv", pool_first=False,
                                          residual_pool=False, depthwise_conv=True, bias_on=True, separate_qkv=True,
                                          embed_dim_mul=None, atten_head_mul=None, dim_mul_in_att=False,
                                          pool_q_stride_size=None, pool_kv_stride_size=None,
                                          pool_kv_stride_adaptive=None, pool_kvq_kernel=None,
                                          head=create_vit_basic_head, head_dropout_rate=0.5, head_activation=None,
                                          head_num_classes=400, create_scriptable_model=False,
                                          multiscale_vit_class=MultiscaleVisionTransformers):
    if use_2d_patch:
        assert temporal_size == 1, "If use_2d_patch, temporal_size needs to be 1."
    if pool_kv_stride_adaptive is not None:
        assert pool_kv_stride_size is None, "pool_kv_stride_size should be none if pool_kv_stride_adaptive is set."
    if norm == "layernorm":
        norm_layer = block_norm_layer = attn_norm_layer = partial(nn.LayerNorm, eps=1e-6)
    elif norm == "batchnorm":
        # BatchNorm1d block norms, BatchNorm3d attention-pool norms (applied before the pool), no final norm
        norm_layer, block_norm_layer, attn_norm_layer = None, nn.BatchNorm1d, nn.BatchNorm3d
    else:
        raise NotImplementedError("Only supports layernorm.")
    if create_scriptable_model and norm == "batchnorm":
        warnings.warn("`create_scriptable_model` is deprecated. MultiscaleVisionTransformers"
                      " now supports scripting without this flag.", DeprecationWarning)
    if isinstance(spatial_size, int):
        spatial_size = (spatial_size, spatial_size)
    patch_embed = create_conv_patch_embed(
        in_channels=input_channels, out_channels=patch_embed_dim, conv_kernel_size=conv_patch_embed_kernel,
        conv_stride=conv_patch_embed_stride, conv_padding=conv_patch_embed_padding,
        conv=nn.Conv2d if use_2d_patch else nn.Conv3d) if enable_patch_embed else None
    in_dims = [temporal_size, spatial_size[0], spatial_size[1]]
    in_stride = (1,) + tuple(conv_patch_embed_stride) if use_2d_patch else conv_patch_embed_stride
    grid = [in_dims[i] // in_stride[i] for i in range(3)] if enable_patch_embed else in_dims
    pos = SpatioTemporalClsPositionalEncoding(embed_dim=patch_embed_dim, patch_embed_shape=grid,
                                              sep_pos_embed=sep_pos_embed, has_cls=cls_embed_on)
    dpr = [x.item() for x in torch.linspace(0, droppath_rate_block, depth)]
    dim_mul, head_mul = torch.ones(depth + 1), torch.ones(depth + 1)
    for i, m in (embed_dim_mul or []):
        dim_mul[i] = m
    for i, m in (atten_head_mul or []):
        head_mul[i] = m
    pool_q = [[] for _ in range(depth)]
    pool_kv = [[] for _ in range(depth)]
    stride_q = [[] for _ in range(depth)]
    stride_kv = [[] for _ in range(depth)]

    def kernel_for(stride):
        return pool_kvq_kernel if pool_kvq_kernel is not None else [s + 1 if s > 1 else s for s in stride]
    for spec in (pool_q_stride_size or []):
        stride_q[spec[0]] = spec[1:]
        pool_q[spec[0]] = kernel_for(spec[1:])
    if pool_kv_stride_adaptive is not None:
        cur = pool_kv_stride_adaptive
        pool_kv_stride_size = []
        for i in range(depth):
            if len(stride_q[i]) > 0:       # K/V stride shrinks whenever Q is pooled
                cur = [max(cur[d] // stride_q[i][d], 1) for d in range(len(cur))]
            pool_kv_stride_size.append([i] + cur)
    for spec in (pool_kv_stride_size or []):
        stride_kv[spec[0]] = spec[1:]
        pool_kv[spec[0]] = kernel_for(spec[1:])

    blocks = nn.ModuleList()
    dim_in = patch_embed_dim
    for i in range(depth):
        num_heads = round_width(num_heads, head_mul[i], min_width=1, divisor=1)
        if dim_mul_in_att:
            dim_out = round_width(dim_in, dim_mul[i], divisor=round_width(num_heads, head_mul[i]))
        else:
            dim_out = round_width(dim_in, dim_mul[i + 1], divisor=round_width(num_heads, head_mul[i + 1]))
        blocks.append(MultiScaleBlock(
            dim=dim_in, dim_out=dim_out, num_heads=num_heads, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias,
            dropout_rate=dropout_rate_block, droppath_rate=dpr[i], norm_layer=block_norm_layer,
            attn_norm_layer=attn_norm_layer,
            dim_mul_in_att=dim_mul_in_att, kernel_q=pool_q[i], kernel_kv=pool_kv[i], stride_q=stride_q[i],
            stride_kv=stride_kv[i], pool_mode=pooling_mode, has_cls_embed=cls_embed_on, pool_first=pool_first,
            residual_pool=residual_pool, bias_on=bias_on, depthwise_conv=depthwise_conv, separate_qkv=separate_qkv))
        dim_in = dim_out
    head_model = head(in_features=dim_in, out_features=head_num_classes,
                      seq_pool_type="cls" if cls_embed_on else "mean", dropout_rate=head_dropout_rate,
                      activation=head_activation) if head is not None else None
    return multiscale_vit_class(patch_embed=patch_embed, cls_positional_encoding=pos,
                                pos_drop=nn.Dropout(p=dropout_rate_block) if dropout_rate_block > 0.0 else None,
                                blocks=blocks, norm_embed=norm_layer(dim_in) if norm_layer else None,
                                head=head_model)
