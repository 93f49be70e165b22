"""Import-only stand-in for the absent `av` (PyAV) package (TEST INFRASTRUCTURE ONLY).

The reference's data/utils.py imports ``av`` and ``av.video.frame.PictureType`` at module load, so its
``pytorchvideo.data`` package cannot be imported without them.  oracle/gen_golden_datasets.py runs only the reference's
frame-folder datasets, which never call PyAV; an encoded-video path fails to load, as a missing decoder would.
"""
