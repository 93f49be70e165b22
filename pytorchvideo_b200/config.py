"""Process-wide defaults for the engine."""
_state = {"precision": "f16", "use_graph": True}


def set_precision(p):
    """'f16' (tensor-core path, f16 storage / fp32 accumulate) or 'f32' (CUDA-core parity mode)."""
    assert p in ("f16", "f32")
    _state["precision"] = p


def get_precision():
    return _state["precision"]


def set_use_graph(flag):
    _state["use_graph"] = bool(flag)


def get_use_graph():
    return _state["use_graph"]
