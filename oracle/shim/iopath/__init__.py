"""Minimal stand-in for the absent `iopath` package (TEST INFRASTRUCTURE ONLY).

The reference's data modules import ``iopath.common.file_io.g_pathmgr`` at module load.  For local paths its
PathManager is the os / builtin file API, which is all oracle/gen_golden_jpeg.py needs to run the reference's
FrameVideo in the authoring container.
"""
