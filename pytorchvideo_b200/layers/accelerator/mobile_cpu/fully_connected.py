import torch.nn as nn

from ....accelerator.no_op_convert_block import NoOpConvertBlock


class FullyConnected(NoOpConvertBlock):
    """nn.Linear(in_features, out_features, bias) as an efficient block (reference
    layers/accelerator/mobile_cpu/fully_connected.py); on its own it takes (batch, tokens, features) inputs."""

    def __init__(self, in_features, out_features, bias=True):
        super().__init__(model=nn.Linear(in_features, out_features, bias=bias))
