"""Soft-target cross entropy (reference losses/soft_target_cross_entropy.py) on the GPU: one launch per call
(pv_soft_target_ce), plus the one-hot conversion of class-index targets.  Forward only: there is no backward."""
import torch
import torch.nn as nn

from .. import contrastive as K
from ..layers.utils import set_attributes
from ..transforms.functional import convert_to_one_hot


class SoftTargetCrossEntropyLoss(nn.Module):
    """Cross entropy against soft (multi-label, MixUp / CutMix) targets: (N, C) logits, (N, C) or (N,) targets.

    ``ignore_index``: as in the reference, a value in [0, C) makes forward raise AttributeError (the reference reads
    the misspelt ``self.ignore_idx``); any other value ignores nothing."""

    def __init__(self, ignore_index: int = -100, reduction: str = "mean", normalize_targets: bool = True) -> None:
        super().__init__()
        set_attributes(self, locals())
        assert isinstance(self.normalize_targets, bool)
        if self.reduction not in ["mean", "none"]:
            raise NotImplementedError('reduction type "{}" not implemented'.format(self.reduction))
        self.eps = torch.finfo(torch.float32).eps

    def forward(self, input: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        if target.ndim == 1:
            assert input.shape[0] == target.shape[0], (
                "SoftTargetCrossEntropyLoss requires input and target to have same batch size!")
            target = convert_to_one_hot(target.reshape(-1), input.shape[1])
        assert input.shape == target.shape, (
            "SoftTargetCrossEntropyLoss requires input and target to be same "
            f"shape: {input.shape} != {target.shape}")
        if input.requires_grad and torch.is_grad_enabled():
            raise RuntimeError("SoftTargetCrossEntropyLoss runs forward only (no backward): call it under torch.no_grad()")
        N, C = target.shape
        if 0 <= self.ignore_index <= C - 1:
            self.ignore_idx          # AttributeError, as the reference's line 63
        # every sample is valid (nothing is ignored), so the mean divides by N
        return K.soft_target_ce(input, target, self.normalize_targets, self.eps, self.reduction)
