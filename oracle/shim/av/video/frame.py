"""``PictureType``: the one name the reference imports from ``av.video.frame``."""
import enum


class PictureType(enum.IntEnum):
    NONE = 0
    I = 1  # noqa: E741
    P = 2
    B = 3
