"""SimCLR (reference models/simclr.py, https://arxiv.org/abs/2002.05709) on the engine: both views through one
[backbone ->] mlp plan, pv_rows_l2_normalize, the second view all-gathered across ranks, and pv_contrastive_ce."""
from typing import Optional

import torch
import torch.distributed as dist
import torch.nn as nn

from .. import contrastive as K
from ..layers.utils import set_attributes
from ..parallel import gather_logits
from .embedding import EmbeddingChain, check_call


class SimCLR(nn.Module):
    """forward(x1, x2) -> the 0-dim fp32 InfoNCE loss of the normalised embeddings at ``temperature``; the target of
    row n is key row ``rank * B + n`` of the gathered second view."""

    def __init__(self, mlp: nn.Module, backbone: Optional[nn.Module] = None, temperature: float = 0.07) -> None:
        super().__init__()
        set_attributes(self, locals())
        self.__dict__["_pv_chain"] = None

    def _chain(self):
        ch = self.__dict__.get("_pv_chain")
        if ch is None or ch.seq[0] is not (self.backbone if self.backbone is not None else self.mlp):
            ch = self.__dict__["_pv_chain"] = EmbeddingChain(self.backbone, self.mlp)
        return ch

    def embed(self, x):
        """F.normalize(mlp(backbone(x)), dim=1) as fp32 (B, C) rows."""
        check_call(self, x)
        return K.l2_normalize(self._chain().embed(x))

    def forward(self, x1: torch.Tensor, x2: torch.Tensor) -> torch.Tensor:
        check_call(self, x1, x2)
        ch = self._chain()
        e1 = K.l2_normalize(ch.embed(x1))
        e2 = K.l2_normalize(ch.embed(x2))
        rank = dist.get_rank() if dist.is_available() and dist.is_initialized() else 0
        keys = gather_logits(e2) if dist.is_available() and dist.is_initialized() else e2
        return K.contrastive_ce(e1, keys, self.temperature, rank * e1.shape[0])
