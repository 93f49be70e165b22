import torch
import torch.nn as nn

from ..module import B200Module
from .efficient_block_base import EfficientBlockBase


class MobileBlock(B200Module, EfficientBlockBase):
    """Base of the mobile efficient blocks (reference layers/accelerator/mobile_cpu/, models/accelerator/mobile_cpu/):
    a parameter container whose forward runs the engine, with the reference's ``convert`` protocol.

    ``convert(input_blob_size)`` keeps the module tree and ``state_dict`` as they are, sets ``convert_flag`` and builds
    the engine's plan for that input shape.  It does not reproduce the reference's deployable form for mobile CPUs
    (Conv3d -> Conv2d decompositions, ``_Reshape``, ``_SkipConnectMul``, the fused ``ConvReLU``): the engine folds
    BatchNorm and fuses activations, residual adds and squeeze-excitation itself.  There is no int8 path, so
    ``convert_for_quantize=True`` raises NotImplementedError."""

    _ALREADY_CONVERTED = "already converted, cannot be converted again"

    def convert(self, input_blob_size, *args, convert_for_quantize=False, native_conv3d_op_qnnpack=False, **kwargs):
        assert self.convert_flag is False, "%s: %s" % (type(self).__name__, self._ALREADY_CONVERTED)
        if convert_for_quantize:
            raise NotImplementedError("%s: quantized (int8) deployment has no engine path" % type(self).__name__)
        self.eval()
        self._pv_compiled(torch.empty(tuple(input_blob_size), dtype=torch.float32, device="cuda"))
        self.convert_flag = True


class NoOpConvertBlock(B200Module, EfficientBlockBase):
    """Wraps ``model`` as an efficient block whose ``convert`` changes nothing
    (reference accelerator/efficient_blocks/no_op_convert_block.py)."""

    def __init__(self, model: nn.Module):
        super().__init__()
        self.model = model

    def convert(self, *args, **kwargs):
        pass
