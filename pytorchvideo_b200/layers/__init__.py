from .swish import Swish  # noqa: F401
from .convolutions import Conv2plus1d, ConvReduce3D, create_conv_2plus1d  # noqa: F401
from .squeeze_excitation import SqueezeExcitation  # noqa: F401
from .utils import round_repeats, round_width, set_attributes  # noqa: F401
from .drop_path import DropPath  # noqa: F401
from .attention import Mlp, MultiScaleAttention, MultiScaleBlock  # noqa: F401,E402
from .positional_encoding import SpatioTemporalClsPositionalEncoding  # noqa: F401,E402
from .positional_encoding import PositionalEncoding  # noqa: F401,E402
from .fusion import ConcatFusion, ReduceFusion, TemporalConcatFusion, make_fusion_layer  # noqa: F401,E402
from .mlp import make_multilayer_perceptron  # noqa: F401,E402
from .batch_norm import NaiveSyncBatchNorm1d, NaiveSyncBatchNorm2d, NaiveSyncBatchNorm3d  # noqa: F401,E402
