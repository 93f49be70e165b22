"""Temperature-scaled contrastive loss (reference pytorchvideo_trainer module/losses.py ``ContrastiveLoss``, MoCo's
objective) on the GPU: cross entropy of inputs / temperature against target 0, one row kernel and the mean
(pv_queue_ce on materialised logits).  contrastive.queue_ce computes the same loss for a query batch against a
key queue without materialising the logits.  Forward only: there is no backward."""
import torch
import torch.nn as nn

from .. import contrastive as K


class ContrastiveLoss(nn.Module):
    def __init__(self, reduction: str = "mean", temperature: float = 0.1) -> None:
        super().__init__()
        if reduction not in ("mean", "none"):
            raise NotImplementedError('reduction type "{}" not implemented'.format(reduction))
        self.reduction = reduction
        self.temperature = temperature

    def forward(self, inputs: torch.Tensor) -> torch.Tensor:
        """inputs: fp32 (N, 1 + K) logits whose column 0 is the positive; the mean loss (0-dim) or the (N,) losses."""
        if inputs.requires_grad and torch.is_grad_enabled():
            raise RuntimeError("ContrastiveLoss runs forward only (no backward): call it under torch.no_grad()")
        return K.logits_ce(inputs, self.temperature, self.reduction)
