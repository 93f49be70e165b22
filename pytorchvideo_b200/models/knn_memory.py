"""The trainer's kNN memory (reference pytorchvideo_trainer module/ssl_helper.py ``KnnMemory``) on the GPU: the
feature bank SSL training writes with ``update`` and val / test score with ``eval_knn``.

``eval_knn`` is two launches of pv_bank_topk (csrc/pv_bank.cu): one scan of the bank per tile of 32 queries keeps each
query's best k similarities per slab without storing the (N, M) similarity matrix, a second launch merges the slabs,
sorts the k neighbours and votes.  ``update`` is one launch of pv_bank_update.  Equal similarities rank the lower bank
index first.  The vote keeps the reference's IEEE arithmetic: a neighbour whose weight exp(sim / T) overflows to +inf
makes every other class of that row NaN (0 * inf), as the reference's one-hot product does.  With the trainer's
settings this is reachable: ``update`` normalises each stored row over a size-1 axis, so every stored value is +-1 and
a unit query's self-similarity is its L1 norm.
"""
import math

import numpy as np
import torch
import torch.nn as nn

from .. import contrastive as K


def _single_process():
    if torch.distributed.is_available() and torch.distributed.is_initialized() and torch.distributed.get_world_size() > 1:
        raise NotImplementedError("KnnMemory on the engine runs in one process: the all_gather of update is not "
                                  "implemented")


class KnnMemory(nn.Module):
    """length x dim bank ``memory`` drawn as the reference draws it (torch.rand on ``device``).  ``eval_knn`` and
    ``update`` run on the GPU only: a bank or labels on the CPU raise RuntimeError."""

    def __init__(self, length: int, dim: int, momentum: float = 1.0, downstream_classes: int = 400,
                 temperature: float = 1.0, knn_k: int = 200, device: str = "cpu") -> None:
        super().__init__()
        self.length = length
        self.dim = dim
        self.momentum = momentum
        self.temperature = temperature
        self.downstream_classes = downstream_classes
        self.knn_k = knn_k
        stdv = 1.0 / math.sqrt(dim / 3)
        self.device = device
        self.register_buffer("memory", torch.rand(length, dim, device=self.device).mul_(2 * stdv).add_(-stdv))

    def resize(self, length: int, dim: int) -> None:
        """A fresh bank of length x dim (as the reference, a plain attribute from here on, no longer a buffer)."""
        self.length = length
        self.dim = dim
        stdv = 1.0 / math.sqrt(dim / 3)
        del self.memory
        self.memory = torch.rand(length, dim, device=self.device).mul_(2 * stdv).add_(-stdv)

    @torch.no_grad()
    def get(self, ind: torch.Tensor) -> torch.Tensor:
        """The bank rows of ``ind`` as (B, -1, dim)."""
        batch_size = ind.size(0)
        return self.memory[ind.view(-1), :].view(batch_size, -1, self.dim)

    def _check_memory(self, x):
        if x.device.type != "cuda":
            raise RuntimeError("pytorchvideo_b200 runs on H100 GPUs only (no CPU path); got a %s tensor" % x.device.type)
        if self.memory.device != x.device:
            raise RuntimeError("the kNN memory is on %s, the features on %s: build KnnMemory with device=%r or move "
                               "the memory with .to()" % (self.memory.device, x.device, str(x.device)))

    @torch.no_grad()
    def update(self, mem: torch.Tensor, ind: torch.Tensor) -> None:
        """memory[ind] = normalize(mem * momentum + memory[ind] * (1 - momentum)) over the reference's size-1 axis,
        i.e. v / max(|v|, 1e-12) elementwise; of repeated indices the last occurrence wins."""
        _single_process()
        self._check_memory(mem)
        x = mem.reshape(mem.size(0), -1)
        K.bank_update(self.memory, x, ind.reshape(-1).to(x.device), self.momentum)

    @torch.no_grad()
    def init_knn_labels(self, train_loader) -> None:
        """The labels of ``train_loader.dataset._labeled_videos`` (host only); resizes the bank to their number."""
        self.num_imgs = len(train_loader.dataset._labeled_videos)
        self.train_labels = np.zeros((self.num_imgs,), dtype=np.int32)
        for i in range(self.num_imgs):
            self.train_labels[i] = train_loader.dataset._labeled_videos[i][1]["label"]
        self.train_labels = torch.LongTensor(self.train_labels).to(self.device)
        if self.length != self.num_imgs:
            self.resize(self.num_imgs, self.dim)

    def forward(self, inputs: torch.Tensor) -> None:
        pass

    @torch.no_grad()
    def eval_knn(self, q_knn: torch.Tensor) -> torch.Tensor:
        """(N, downstream_classes) fp32 votes of the knn_k nearest bank rows (similarity q . m) of each query row."""
        labels = self.train_labels                         # AttributeError before init_knn_labels, as the reference
        self._check_memory(q_knn)
        if labels.device != q_knn.device:
            raise RuntimeError("the kNN labels are on %s, the features on %s: build KnnMemory with device=%r (the "
                               "labels go to self.device) or move them with .to()" % (labels.device, q_knn.device,
                                                                                      str(q_knn.device)))
        q = q_knn.reshape(q_knn.size(0), -1)
        memory = self.memory.reshape(self.memory.size(0), -1)
        _, _, preds = K.bank_topk(q, memory, self.knn_k, labels, self.downstream_classes, self.temperature)
        return preds
