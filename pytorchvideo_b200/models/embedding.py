"""The embedding path of the self-supervised models: [backbone] -> [projector / predictor] as ONE engine plan.

``EmbeddingChain`` holds the modules of a wrapper (``SimCLR``, ``BYOL``, ``MemoryBank``) without registering them a
second time: it lives in the wrapper's ``__dict__``, so the wrapper's module tree and state_dict keys stay the
reference's.  It lowers as an nn.Sequential of its parts (engine/lower.py): a headless ResNet trunk pools to (B, C)
rows and every Linear -> [BatchNorm] -> [ReLU] of the projector is one GEMM launch.  The result is fp32 (B, C) rows."""
import torch
import torch.nn as nn

from ..module import B200Module


class EmbeddingChain(B200Module):
    def __init__(self, *parts):
        super().__init__()
        self.seq = nn.Sequential(*[p for p in parts if p is not None])
        self.training = False

    def train(self, mode=True):
        # the chain never trains and leaves the shared modules' flags alone; the wrapper checks its own mode
        self.training = False
        return self

    def embed(self, x):
        if not torch.is_tensor(x):
            raise RuntimeError("expected a tensor input")
        return self(x)


def _lower_embedding_chain(self, m, x, name):
    self.fuse_rows = True
    try:
        return self.lower_Sequential(m.seq, x, name or "seq")
    finally:
        self.fuse_rows = False


def _register():
    from ..engine.lower import Lowering
    Lowering.lower_EmbeddingChain = _lower_embedding_chain


_register()


def check_call(wrapper, *xs):
    """The engine's rules for a wrapper's forward: eval mode and CUDA inputs."""
    if wrapper.training:
        raise RuntimeError("pytorchvideo_b200 is an eval-mode forward engine: call model.eval() first")
    for x in xs:
        if not torch.is_tensor(x):
            raise RuntimeError("expected tensor inputs")
        if x.device.type != "cuda":
            raise RuntimeError("pytorchvideo_b200 runs on H100 GPUs only (no CPU path); got a %s tensor" % x.device.type)
