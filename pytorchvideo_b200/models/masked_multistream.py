"""Modules that take a tensor and a mask (reference models/masked_multistream.py:35-384): how a long video, a
variable-length sequence of clip features, is classified and fused across streams.

Every class is a parameter container with the reference's constructor, attribute names, ``state_dict`` keys and
``repr``; its forward runs on the engine (engine/lower.py, the ``masked`` lowerings).  A mask is a bool
``(batch_size, seq_len)`` tensor, ``False`` marking an invalid step; ``mask=None`` compiles a plan of its own in which
every step is valid.  The mask enters the plan as u8 data, so one compiled plan (and its CUDA graph) serves every mask
of one shape.

Deviations from the reference, all on purpose:

- Caller tensors are never mutated.  The reference's ``TransposeMultiheadAttention`` and ``TransposeTransformerEncoder``
  set ``mask[:, 0] = True`` on the mask they receive, and ``MaskedTemporalPooling("max")`` writes ``-inf`` / ``0`` into
  the caller's ``x``.  The engine applies the forced first column to the plan's own copy of the mask, so the modules
  after an attention module inside a ``MaskedSequential`` (or one stream of a ``MaskedMultiPathWay``) see it exactly as
  they do in the reference, while the caller's mask keeps its values.
  Each stream of a ``MaskedMultiPathWay`` has its own copy: when a caller passes one mask object to several streams,
  the reference's write also reaches the streams after the first attention module's; the engine's does not.
- ``MaskedMultiPathWay`` without a fusion raises ``RuntimeError``; the reference fails with ``UnboundLocalError``.
"""
from typing import List, Optional, Tuple

import torch
import torch.nn as nn

from ..layers.utils import set_attributes
from ..module import B200Module


class _MaskedModule(B200Module):
    """forward(x, mask) through the engine; ``attention_weights`` of nested ``TransposeMultiheadAttention`` modules are
    copied out of the plan after every call."""

    def _pv_masked(self, pairs, multi=False):
        ins, has = [], []
        for x, mask in pairs:
            if not torch.is_tensor(x):
                raise RuntimeError("expected a tensor input, got %s" % type(x).__name__)
            ins.append(x)
            if mask is not None:
                if not torch.is_tensor(mask) or mask.dtype != torch.bool:
                    raise RuntimeError("mask must be a bool tensor, got %s" % (
                        mask.dtype if torch.is_tensor(mask) else type(mask).__name__))
                if mask.dim() != 2 or mask.shape[0] != x.shape[0]:
                    raise RuntimeError("mask of shape %s is not a (batch_size, seq_len) mask for x of shape %s" % (
                        tuple(mask.shape), tuple(x.shape)))
                ins.append(mask)
            has.append(mask is not None)
        cm = self._pv_compiled(ins, extra=(("masks", bool(multi)) + tuple(has),))
        out = cm(ins).clone()
        for module, tensor, shape in cm.side_outputs():
            module._attention_weights = tensor.clone().view(shape)
        return out


class MaskedTemporalPooling(_MaskedModule):
    """Pools (batch_size, seq_len, feature_dim) over the valid steps: "max" (a row with no valid step gives 0), "avg"
    (masked sum / max(valid count, 1)) or "sum"; fp32 accumulation."""

    def __init__(self, method: str):
        super().__init__()
        assert method in ("max", "avg", "sum")
        self._method = method

    def forward(self, x: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        return self._pv_masked([(x, mask)])


class TransposeMultiheadAttention(_MaskedModule):
    """nn.MultiheadAttention over (batch_size, seq_len, feature_dim) with the mask as key padding mask (column 0 forced
    valid).  ``attention_weights`` holds the head-averaged (batch_size, seq_len, seq_len) fp32 softmax of the last
    call, as with ``need_weights=True``."""

    def __init__(self, feature_dim: int, num_heads: int = 1):
        super().__init__()
        self._attention = nn.MultiheadAttention(embed_dim=feature_dim, num_heads=num_heads)
        self._attention_weights = None

    @property
    def attention_weights(self) -> Optional[torch.Tensor]:
        """Contains attention weights from last forward call."""
        return self._attention_weights

    def forward(self, x: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        return self._pv_masked([(x, mask)])


class LearnMaskedDefault(_MaskedModule):
    """x * any(mask) + default * (1 - any(mask)) in fp32: rows without any valid step get the learned default."""

    def __init__(self, feature_dim: int, init_method: str = "gaussian", freeze: bool = False):
        super().__init__()
        if init_method == "zeros":
            self._learned_defaults = nn.Parameter(torch.zeros(feature_dim), requires_grad=(not freeze))
        elif init_method == "gaussian":
            self._learned_defaults = nn.Parameter(torch.Tensor(feature_dim), requires_grad=(not freeze))
            nn.init.normal_(self._learned_defaults)
        else:
            raise NotImplementedError(f"{init_method} not available. Options are: 'zeros' or 'gaussian'")

    def forward(self, x: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
        if mask is None:
            raise RuntimeError("LearnMaskedDefault.forward needs a mask")
        return self._pv_masked([(x, mask)])


class LSTM(_MaskedModule):
    """Masked LSTM (``nn.LSTM`` with ``batch_first=True`` as the parameter holder): row b runs its first
    clamp(mask[b].sum(), 1, seq_len) steps; the output is h_n, cat(forward, reverse) when bidirectional."""

    def __init__(self, dim_in: int, hidden_dim: int, dropout: float = 0.0, bidirectional: bool = False):
        super().__init__()
        self.lstm = nn.LSTM(dim_in, hidden_dim, batch_first=True, dropout=dropout, bidirectional=bidirectional)
        self.lstm.flatten_parameters()
        self.output_dim = 2 * hidden_dim if bidirectional else hidden_dim
        self.bidirectional = bidirectional

    def forward(self, data: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        return self._pv_masked([(data, mask)])


class TransposeTransformerEncoder(_MaskedModule):
    """nn.TransformerEncoder (post-norm layers, ReLU, dim_feedforward 2048) with the mask as key padding mask (column 0
    forced valid); returns the sequence's first position, (batch_size, feature_dim)."""

    def __init__(self, dim_in: int, num_heads: int = 1, num_layers: int = 1):
        super().__init__()
        self.encoder = nn.TransformerEncoder(nn.TransformerEncoderLayer(dim_in, num_heads), num_layers)

    def forward(self, data: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        return self._pv_masked([(data, mask)])


class MaskedSequential(_MaskedModule, nn.Sequential):
    """Sequential container whose mask modules (the classes above) receive the mask; every other member gets the
    tensor alone."""

    _MASK_MODULES = [MaskedTemporalPooling, LearnMaskedDefault, TransposeMultiheadAttention, LSTM,
                     TransposeTransformerEncoder]

    def forward(self, input: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
        return self._pv_masked([(input, mask)])


class MaskedMultiPathWay(_MaskedModule):
    """One masked stream per pathway, then a fusion of their outputs.  ``multipathway_fusion=None`` raises
    ``RuntimeError`` at forward (the reference fails with ``UnboundLocalError``)."""

    def __init__(self, *, multipathway_blocks: nn.ModuleList, multipathway_fusion: Optional[nn.Module]) -> None:
        super().__init__()
        set_attributes(self, locals())

    def forward(self, x_and_mask: List[Tuple[torch.Tensor, torch.Tensor]]) -> torch.Tensor:
        if self.multipathway_fusion is None:
            raise RuntimeError("MaskedMultiPathWay needs a multipathway_fusion to reduce its streams")
        if len(x_and_mask) != len(self.multipathway_blocks):
            raise RuntimeError("expected %d (x, mask) pairs, got %d" % (len(self.multipathway_blocks), len(x_and_mask)))
        return self._pv_masked([tuple(p) for p in x_and_mask], multi=True)
