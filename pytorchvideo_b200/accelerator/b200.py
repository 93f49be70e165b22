""""b200" target: wraps a supported block (this package's or the reference's own module - the
lowering dispatches on class/attribute names) into an EfficientBlockBase whose ``convert`` builds
the static plan + CUDA graph for the recorded input shape."""
from copy import deepcopy

import torch
import torch.nn as nn

from .efficient_block_base import EfficientBlockBase
from .model_transmuter import EFFICIENT_BLOCK_TRANSMUTER_REGISTRY, transmute_model

_WHOLE_BLOCKS = ("Net", "ResStage", "ResBlock", "BottleneckBlock", "ResNetBasicStem", "ResNetBasicHead",
                 "MultiPathWayWithFuse", "ProjectedPool", "NonLocal", "EfficientX3d", "X3dBottleneckBlock")


class B200Block(EfficientBlockBase):
    def __init__(self, block: nn.Module, dtype="f16"):
        super().__init__()
        self.block = block            # parameters stay owned by the original module (same state_dict keys + "block.")
        self.dtype = dtype
        self._compiled = None         # the plan built by convert(input_blob_size)
        self._by_shape = {}           # further shapes seen at run time (a final partial batch): one plan each

    @staticmethod
    def _shapes(x):
        return tuple(tuple(t.shape) for t in x) if isinstance(x, (list, tuple)) else (tuple(x.shape),)

    def _compile(self, shapes, device="cuda"):
        from ..engine import compile_model
        ex = [torch.empty(tuple(s), dtype=torch.float32, device=device) for s in shapes]
        self.block.eval()
        return compile_model(self.block, ex if len(ex) > 1 else ex[0], dtype=self.dtype)

    def convert(self, input_blob_size=None, **kwargs):
        """EfficientBlockBase protocol (efficient_block_base.py:8-35): build the deployable form for the given input
        size - here the static plan (BN folded, weights re-laid-out, TMA descriptors, CUDA graph).  Like the
        reference's mobile blocks (convolutions.py:120-122) a block converts once."""
        assert self._compiled is None, "B200Block: already converted, cannot be converted again"
        if input_blob_size is None:
            raise ValueError("convert() needs the input shape(s)")
        shapes = tuple(tuple(s) for s in input_blob_size) if isinstance(input_blob_size[0], (tuple, list, torch.Size)) \
            else (tuple(input_blob_size),)
        self._compiled = self._compile(shapes)
        self._by_shape[shapes] = self._compiled

    def forward(self, x):
        shapes = self._shapes(x)
        cm = self._by_shape.get(shapes)
        if cm is None:                # unconverted block, or a shape convert() was not given: one more plan
            dev = (x[0] if isinstance(x, (list, tuple)) else x).device
            cm = self._by_shape[shapes] = self._compile(shapes, dev)
            if self._compiled is None:
                self._compiled = cm
        return cm(x).clone()


def transmute_b200(module: nn.Module):
    """Transmuter fn: returns a B200Block for whole blocks the engine can lower, else None."""
    if type(module).__name__ in _WHOLE_BLOCKS:
        return B200Block(module)
    return None


EFFICIENT_BLOCK_TRANSMUTER_REGISTRY.setdefault("b200", []).append(transmute_b200)


def convert_to_deployable_form(model: nn.Module, input_tensor, whole_model=True, **kwargs) -> nn.Module:
    """Reference protocol (mobile_cpu/utils/model_conversion.py:87-125): deep-copy, eval, record each
    efficient block's input shape with one hooked forward, then call ``convert(input_blob_size)``.

    A model that was already transmuted (``transmute_model(model, "b200")``) keeps its blocks.  An untouched model
    that the engine can lower as a whole becomes ONE block (one plan, no NCDHW round trips between blocks);
    ``whole_model=False`` forces the per-block route of the reference protocol."""
    model = deepcopy(model).eval()
    transmuted = any(isinstance(m, B200Block) for m in model.modules())
    if not transmuted and whole_model and type(model).__name__ in _WHOLE_BLOCKS:
        model = B200Block(model)
        shapes = [tuple(t.shape) for t in input_tensor] if isinstance(input_tensor, (list, tuple)) else tuple(input_tensor.shape)
        model.convert(shapes)
        return model
    if not transmuted:
        transmute_model(model, "b200")
    # one hooked forward: every efficient block is converted, explicitly, with the input size it actually receives
    # (model_conversion.py:104-123 records input_blob_size the same way, then calls convert on each block)
    hooks = []
    for m in model.modules():
        if isinstance(m, B200Block):
            def hook(mod, inp):
                if mod._compiled is None:
                    mod.convert(B200Block._shapes(inp[0]) if isinstance(inp[0], (list, tuple)) else tuple(inp[0].shape))
            hooks.append(m.register_forward_pre_hook(hook))
    with torch.no_grad():
        model(input_tensor)
    for h in hooks:
        h.remove()
    return model
