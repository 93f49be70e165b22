"""Non-local block (reference layers/nonlocal_net.py:10-155): the long-range attention block of the I3D-NLN and
SlowFast+NL models.  ``NonLocal`` is a parameter container with the reference's constructor and attribute names;
its forward runs on the engine (engine/lower.py ``lower_NonLocal``): the theta / phi / g projections as token GEMMs,
the optional max pool, one single-head flash attention of width ``dim_inner`` (softmax or "dot_product"), and
``conv_out`` with the norm folded and the identity residual fused into its epilogue."""
from typing import Callable, Iterable, Optional, Tuple

import torch.nn as nn

from ..module import B200Module
from .utils import set_attributes


class NonLocal(B200Module):
    """x + norm(conv_out(A(theta(x), phi(pool(x))) g(pool(x)))) with A = softmax(theta^T phi / sqrt(dim_inner))
    ("softmax") or theta^T phi / N_k ("dot_product", N_k = positions after the pool)."""

    def __init__(self, *, conv_theta: nn.Module, conv_phi: nn.Module, conv_g: nn.Module, conv_out: nn.Module,
                 pool: Optional[nn.Module] = None, norm: Optional[nn.Module] = None,
                 instantiation: str = "dot_product") -> None:
        super().__init__()
        set_attributes(self, locals())
        assert None not in (conv_theta, conv_phi, conv_g, conv_out)
        assert instantiation in ("dot_product", "softmax"), "Unknown norm type {}".format(instantiation)
        assert len({self.conv_theta.out_channels, self.conv_phi.out_channels, self.conv_g.out_channels,
                    self.conv_out.in_channels}) == 1, "Nonlocal convolution's input/ output dimension mismatch."


def create_nonlocal(*, dim_in: int, dim_inner: int, pool_size: Optional[Tuple[int]] = (1, 1, 1),
                    instantiation: str = "softmax", norm: Optional[Callable] = nn.BatchNorm3d, norm_eps: float = 1e-5,
                    norm_momentum: float = 0.1):
    """Reference nonlocal_net.py:98-155: 1x1x1 theta / phi / g / out convolutions with bias, a MaxPool3d with
    kernel = stride = ``pool_size`` when some size is > 1, and ``norm(dim_in)`` after conv_out."""
    if pool_size is None:
        pool_size = (1, 1, 1)
    assert isinstance(pool_size, Iterable)
    norm_model = None if norm is None else norm(num_features=dim_in, eps=norm_eps, momentum=norm_momentum)
    if any(size > 1 for size in pool_size):
        pool_model = nn.MaxPool3d(kernel_size=pool_size, stride=pool_size, padding=[0, 0, 0])
    else:
        pool_model = None
    return NonLocal(
        conv_theta=nn.Conv3d(dim_in, dim_inner, kernel_size=1, stride=1, padding=0),
        conv_phi=nn.Conv3d(dim_in, dim_inner, kernel_size=1, stride=1, padding=0),
        conv_g=nn.Conv3d(dim_in, dim_inner, kernel_size=1, stride=1, padding=0),
        conv_out=nn.Conv3d(dim_inner, dim_in, kernel_size=1, stride=1, padding=0),
        pool=pool_model,
        norm=norm_model,
        instantiation=instantiation,
    )
