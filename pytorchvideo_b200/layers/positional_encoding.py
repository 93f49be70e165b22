"""Positional encodings: the sinusoidal ``PositionalEncoding`` (reference layers/positional_encoding.py:11-44) and the
cls token + separable spatio-temporal positional encoding container (:47-136)."""
import math
from typing import Tuple

import torch
import torch.nn as nn

from ..module import B200Module


class PositionalEncoding(B200Module):
    """x + pe[:, :seq_len, :] on (batch_size, seq_len, embed_dim) tokens, PE(pos, 2i) = sin(pos / 10000^(2i/d)),
    PE(pos, 2i+1) = cos(...); the ``pe`` buffer is built as the reference builds it.  On device one add launch
    (pv_add_pos_cls without a cls token)."""

    def __init__(self, embed_dim: int, seq_len: int = 1024) -> None:
        super().__init__()
        pe = torch.zeros(seq_len, embed_dim, dtype=torch.float)
        position = torch.arange(0, seq_len, dtype=torch.float).unsqueeze(1)
        div_term = torch.exp(torch.arange(0, embed_dim, 2).float() * (-(math.log(10000.0)) / embed_dim))
        pe[:, 0::2] = torch.sin(position * div_term)
        pe[:, 1::2] = torch.cos(position * div_term)
        pe = pe.unsqueeze(0)
        self.register_buffer("pe", pe)


class SpatioTemporalClsPositionalEncoding(B200Module):
    """Parameters: cls_token, pos_embed_spatial [1,HW,C], pos_embed_temporal [1,T,C],
    pos_embed_class [1,1,C] (or one pos_embed when sep_pos_embed=False).  On device the engine adds
    spatial[i % HW] + temporal[i // HW] to patch token i and prepends cls_token + pos_embed_class."""

    def __init__(self, embed_dim: int, patch_embed_shape: Tuple[int, int, int], sep_pos_embed: bool = False,
                 has_cls: bool = True) -> None:
        super().__init__()
        assert len(patch_embed_shape) == 3, "Patch_embed_shape should be in the form of (T, H, W)."
        self.cls_embed_on = has_cls
        self.sep_pos_embed = sep_pos_embed
        self._patch_embed_shape = tuple(patch_embed_shape)
        self.num_spatial_patch = patch_embed_shape[1] * patch_embed_shape[2]
        self.num_temporal_patch = patch_embed_shape[0]
        n = self.num_spatial_patch * self.num_temporal_patch
        if has_cls:
            self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
            n += 1
        else:
            self.cls_token = torch.tensor(0)
        if sep_pos_embed:
            self.pos_embed_spatial = nn.Parameter(torch.zeros(1, self.num_spatial_patch, embed_dim))
            self.pos_embed_temporal = nn.Parameter(torch.zeros(1, self.num_temporal_patch, embed_dim))
            self.pos_embed_class = nn.Parameter(torch.zeros(1, 1, embed_dim)) if has_cls else torch.tensor([])
            self.pos_embed = torch.tensor([])
        else:
            self.pos_embed = nn.Parameter(torch.zeros(1, n, embed_dim))
            self.pos_embed_spatial = torch.tensor([])
            self.pos_embed_temporal = torch.tensor([])
            self.pos_embed_class = torch.tensor([])

    def patch_embed_shape(self) -> Tuple[int, int, int]:
        return self._patch_embed_shape
