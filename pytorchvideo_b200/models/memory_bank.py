"""Non-parametric instance discrimination with a memory bank (reference models/memory_bank.py,
https://arxiv.org/abs/1805.01978) on the engine: backbone [-> mlp] as one plan, pv_rows_l2_normalize, the reference's
host draw of the negative indices, and pv_memory_bank_ce, which gathers the K = neg_size + 1 bank rows of every sample
and reduces their logits without materialising the (B, K, dim) gather."""
import math
from typing import Optional

import torch
import torch.nn as nn

from .. import contrastive as K
from ..layers.utils import set_attributes
from .embedding import EmbeddingChain, check_call


class MemoryBank(nn.Module):
    """forward(x, x_ind) -> the 0-dim fp32 loss.  Eval only: the training-mode bank update is not implemented, so
    training mode raises RuntimeError like every engine forward.  The bank is a ``memory`` buffer of shape
    (bank_size, dim), drawn as the reference does (one torch.rand call on the CPU: 10 GB of host memory at the
    defaults)."""

    def __init__(self, backbone: nn.Module, mlp: Optional[nn.Module] = None, neg_size: int = 4096,
                 temperature: float = 0.07, bank_size: int = 1280000, dim: int = 2048, mmt: float = 0.999) -> None:
        super().__init__()
        set_attributes(self, locals())
        self._init_mem_bank(bank_size, dim)
        self.__dict__["_pv_chain"] = None

    def _init_mem_bank(self, bank_size: int, dim: int) -> None:
        stdv = 1.0 / math.sqrt(dim / 3)
        self.register_buffer(
            "memory",
            torch.rand(bank_size, dim).mul_(2 * stdv).add_(-stdv).to(next(self.backbone.parameters()).device))

    def _chain(self):
        ch = self.__dict__.get("_pv_chain")
        if ch is None or ch.seq[0] is not self.backbone:
            ch = self.__dict__["_pv_chain"] = EmbeddingChain(self.backbone, self.mlp)
        return ch

    def embed(self, x):
        """F.normalize([mlp](backbone(x)), dim=1) as fp32 (B, dim) rows."""
        check_call(self, x)
        return K.l2_normalize(self._chain().embed(x))

    def draw_indices(self, batch_size, x_ind, device):
        """The reference's draw (memory_bank.py:92-96): torch.randint(0, bank_size, (B, neg_size + 1)) on torch's CPU
        generator, moved to ``device``, with column 0 replaced by ``x_ind``."""
        idx = torch.randint(0, self.bank_size, size=(batch_size, self.neg_size + 1)).to(device)
        idx.select(1, 0).copy_(x_ind.data)
        return idx

    def forward(self, x: torch.Tensor, x_ind: torch.Tensor) -> torch.Tensor:
        check_call(self, x)
        if self.memory.device != x.device:
            raise RuntimeError("the memory bank is on %s, the input on %s: move the model with .to()" % (
                self.memory.device, x.device))
        if self.memory.dtype != torch.float32:
            raise RuntimeError("the memory bank must be float32, not %s" % self.memory.dtype)
        batch_size = x.shape[0]
        if not torch.is_tensor(x_ind) or x_ind.numel() != batch_size:
            raise RuntimeError("x_ind must hold one bank index per sample")
        e = K.l2_normalize(self._chain().embed(x))
        idx = self.draw_indices(batch_size, x_ind, x.device)
        return K.memory_bank_ce(e, self.memory, idx, self.temperature)
