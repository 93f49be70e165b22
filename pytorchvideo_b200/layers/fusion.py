"""Fusion layers (reference layers/fusion.py:17-149): reduce a list of (batch_size, seq_len, feature_dim) stream
outputs - or (batch_size, feature_dim) pooled ones - to one tensor.  Parameter-free containers with the reference's
constructors; the forward runs on the engine (engine/lower.py): ``ConcatFusion`` as channel-slice writes of the
producers into one buffer, ``TemporalConcatFusion`` as row copies, ``ReduceFusion`` as one elementwise
max / sum / prod launch.  ``ReduceFusion``'s ``reduce_fn`` is classified on the host (engine/lower.py
``reduce_fusion_op``); another function raises ``NotImplementedError``."""
from typing import Callable, List

import torch

from ..module import B200Module


def make_fusion_layer(method: str, feature_dims: List[int]):
    """method: 'concat', 'temporal_concat', 'max', 'sum' or 'prod'; feature_dims: the feature_dim of every input."""
    if method == "concat":
        return ConcatFusion(feature_dims)
    elif method == "temporal_concat":
        return TemporalConcatFusion(feature_dims)
    elif method == "max":
        return ReduceFusion(feature_dims, lambda x: torch.max(x, dim=0).values)
    elif method == "sum":
        return ReduceFusion(feature_dims, lambda x: torch.sum(x, dim=0))
    elif method == "prod":
        return ReduceFusion(feature_dims, lambda x: torch.prod(x, dim=0))
    else:
        raise NotImplementedError(f"Fusion {method} not available.")


class _Fusion(B200Module):
    def forward(self, input_list: List[torch.Tensor]) -> torch.Tensor:
        if not isinstance(input_list, (list, tuple)) or not input_list:
            raise RuntimeError("a fusion layer takes a non-empty list of tensors")
        return super().forward(list(input_list))


class ConcatFusion(_Fusion):
    """torch.cat(input_list, dim=-1)."""

    def __init__(self, feature_dims: List[int]):
        super().__init__()
        _verify_feature_dim(feature_dims)
        self._output_dim = sum(feature_dims)

    @property
    def output_dim(self):
        """Last dimension size of forward(..) tensor output."""
        return self._output_dim


class TemporalConcatFusion(_Fusion):
    """torch.cat(input_list, dim=1)."""

    def __init__(self, feature_dims: List[int]):
        super().__init__()
        _verify_feature_dim(feature_dims)
        self._output_dim = max(feature_dims)
        assert self._output_dim == min(feature_dims)

    @property
    def output_dim(self):
        """Last dimension size of forward(..) tensor output."""
        return self._output_dim


class ReduceFusion(_Fusion):
    """reduce_fn(torch.stack(input_list)) for reduce_fn = max / sum / prod over dim 0."""

    def __init__(self, feature_dims: List[int], reduce_fn: Callable[[torch.Tensor], torch.Tensor]):
        super().__init__()
        _verify_feature_dim(feature_dims)
        self.reduce_fn = reduce_fn
        self._output_dim = max(feature_dims)
        assert self._output_dim == min(feature_dims)

    @property
    def output_dim(self):
        """Last dimension size of forward(..) tensor output."""
        return self._output_dim


def _verify_feature_dim(feature_dims: List[int]):
    assert isinstance(feature_dims, list)
    assert all(x > 0 for x in feature_dims)
