from .soft_target_cross_entropy import SoftTargetCrossEntropyLoss  # noqa: F401
from .contrastive_loss import ContrastiveLoss  # noqa: F401
