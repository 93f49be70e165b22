"""Base class of every block in this package: a parameter container whose ``forward`` runs the
B200 engine.  There is no ATen / CPU forward: calling a block with CPU tensors, in training mode
or without the CUDA library raises."""
import torch
import torch.nn as nn

from . import config


class B200Module(nn.Module):
    _PV_CACHE_PLANS = 4      # compiled plans kept per module (LRU): alternating shapes do not re-capture a graph

    def _pv_fingerprint(self):
        """Cheap change detector for the derived weight copies: in-place updates (load_state_dict,
        optimizer steps) bump ``_version``; ``.to()`` / ``.cuda()`` move the storage.  The list of
        tensors is collected once - Parameter / buffer OBJECTS survive both kinds of update."""
        ts = self.__dict__.get("_pv_tensors")
        if ts is None:
            ts = [t for t in self.parameters()] + [t for t in self.buffers()]
            self.__dict__["_pv_tensors"] = ts
        v = len(ts)
        for t in ts:
            v += t._version + (t.data_ptr() & 0xFFFFF)
        return v

    def _pv_compiled(self, x, extra=()):
        from .engine import compile_model
        ins = x if isinstance(x, (list, tuple)) else [x]
        for t in ins:
            if not torch.is_tensor(t):
                raise RuntimeError("expected tensor inputs")
            if t.device.type != "cuda":
                raise RuntimeError(
                    "pytorchvideo_b200 runs on H100 GPUs only (no CPU path); got a %s tensor" % t.device.type)
        if self.training:
            raise RuntimeError("pytorchvideo_b200 is an eval-mode forward engine: call model.eval() first")
        key = (tuple((tuple(t.shape), t.dtype, t.device.index) for t in ins), config.get_precision(),
               config.get_use_graph(), tuple(extra), self._pv_fingerprint())
        cache = self.__dict__.setdefault("_pv_cache", {})
        cm = cache.pop(key, None)
        if cm is None:
            fp = key[-1]
            for k in [k for k in cache if k[-1] != fp]:
                del cache[k]                       # weights changed: every older plan holds stale packed copies
            while len(cache) >= self._PV_CACHE_PLANS:
                del cache[next(iter(cache))]       # least recently used
            cm = compile_model(self, list(ins) if isinstance(x, (list, tuple)) else x, config.get_precision(),
                               config.get_use_graph(), extra=extra)
        cache[key] = cm                            # (re)insert at the most-recently-used end
        return cm

    def __getstate__(self):
        """copy.deepcopy / pickle (the reference's transmuter deep-copies the model): compiled plans hold device
        buffers, CUDA graphs and ctypes descriptors and are derived data - a copy recompiles on its first call."""
        st = dict(self.__dict__)
        st.pop("_pv_cache", None)
        st.pop("_pv_tensors", None)
        return st

    def _apply(self, fn, *a, **k):
        self.__dict__.pop("_pv_tensors", None)     # .to()/.cuda() may replace parameter objects
        return super()._apply(fn, *a, **k)

    def forward(self, x, *extra):
        """``extra``: non-tensor forward arguments (MViT blocks: ``thw_shape``).  Modules with a second,
        host-side result (the pooled thw) return ``(tensor, aux)`` like the reference."""
        extra = tuple(tuple(int(v) for v in e) if isinstance(e, (list, tuple)) else e for e in extra)
        cm = self._pv_compiled(x, extra)
        out = cm(x).clone()
        return out if cm.aux is None else (out, list(cm.aux))
