"""Multi-layer perceptron builder (reference layers/mlp.py): the projector / predictor of the self-supervised models.
The engine lowers each Linear -> [norm] -> [ReLU] of it on (B, C) rows as one GEMM launch (engine/lower.py)."""
from typing import Callable, List, Optional, Tuple

from torch import nn


def make_multilayer_perceptron(
    fully_connected_dims: List[int],
    norm: Optional[Callable] = None,
    mid_activation: Callable = nn.ReLU,
    final_activation: Optional[Callable] = nn.ReLU,
    dropout_rate: float = 0.0,
) -> Tuple[nn.Module, int]:
    """Linear(fc[i-1], fc[i]) -> norm -> mid_activation for every inner width, then Linear to fc[-1], Dropout (when
    dropout_rate > 0) and final_activation.  Returns (nn.Sequential, fc[-1]) with the reference's module tree."""
    assert isinstance(fully_connected_dims, list)
    assert len(fully_connected_dims) > 1
    assert all(_is_pos_int(x) for x in fully_connected_dims)

    layers = []
    cur_dim = fully_connected_dims[0]
    for dim in fully_connected_dims[1:-1]:
        layers.append(nn.Linear(cur_dim, dim))
        if norm is not None:
            layers.append(norm(dim))
        layers.append(mid_activation())
        cur_dim = dim
    layers.append(nn.Linear(cur_dim, fully_connected_dims[-1]))
    if dropout_rate > 0:
        layers.append(nn.Dropout(p=dropout_rate))
    if final_activation is not None:
        layers.append(final_activation())
    return nn.Sequential(*layers), fully_connected_dims[-1]


def _is_pos_int(number: int) -> bool:
    """True for an int >= 0: like the reference, 0 passes (nn.Linear then has an empty side)."""
    return type(number) == int and number >= 0
