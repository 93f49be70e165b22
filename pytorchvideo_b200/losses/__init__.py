from .soft_target_cross_entropy import SoftTargetCrossEntropyLoss  # noqa: F401
