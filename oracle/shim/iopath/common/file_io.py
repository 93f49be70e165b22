"""``g_pathmgr`` for local paths only: isdir, isfile, ls, open, exists, as iopath's native handler does them."""
import os


class _LocalPathManager:
    def isdir(self, path):
        return os.path.isdir(path)

    def isfile(self, path):
        return os.path.isfile(path)

    def exists(self, path):
        return os.path.exists(path)

    def ls(self, path):
        return os.listdir(path)

    def open(self, path, mode="r", **kwargs):
        return open(path, mode, **kwargs)


g_pathmgr = _LocalPathManager()
PathManager = _LocalPathManager
