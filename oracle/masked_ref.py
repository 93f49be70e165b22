"""Restatement of the masked multistream forward (models/masked_multistream.py, layers/fusion.py,
layers/positional_encoding.py:11-44) in plain torch on the CPU, at any floating dtype (float64 for the kernel tests).

Dispatch is by class name and attribute names, so it runs this package's module trees and the reference's alike.
Nothing is written into the caller's tensors: the forced first mask column of the attention modules is applied to a
copy that the later modules of the same stream receive, which is what the reference's in-place write amounts to.
Returns (output, {module path: head-averaged attention weights}).
"""
import torch
import torch.nn.functional as F

_MASK_MODULES = ("MaskedTemporalPooling", "LearnMaskedDefault", "TransposeMultiheadAttention", "LSTM",
                 "TransposeTransformerEncoder")


def _p(t, dt):
    return None if t is None else t.detach().to(dt)


def _pool(m, x, mask):
    b, t = x.shape[0], x.shape[1]
    if mask is None:
        mask = torch.ones((b, t), dtype=torch.bool)
    if m._method == "max":
        x = x.clone()
        x[~mask, :] = float("-inf")
        x[~mask.view(b, -1).any(dim=-1), :] = 0
        return torch.max(x, dim=1)[0]
    x = (x * mask.unsqueeze(-1).to(x.dtype)).sum(dim=1)
    if m._method == "sum":
        return x
    n = mask.view(b, t, -1).any(dim=-1).to(x.dtype).sum(dim=-1).int()
    return x.div(n.clamp(min=1).unsqueeze(-1).expand(x.size()).to(x.dtype))


def _default(m, x, mask):
    a = mask.view(mask.shape[0], -1).any(dim=-1)
    for i in range(1, x.dim()):
        a = a.unsqueeze(i)
    a = a.to(x.dtype)
    return x * a + _p(m._learned_defaults, x.dtype) * (1 - a)


def _mha(a, x, key_valid, dt):
    """nn.MultiheadAttention(x, x, x, key_padding_mask=~key_valid) on (B, T, E): (output, head-averaged weights)."""
    B, T, E = x.shape
    H = a.num_heads
    D = E // H
    qkv = F.linear(x, _p(a.in_proj_weight, dt), _p(a.in_proj_bias, dt))
    q, k, v = (qkv[..., i * E:(i + 1) * E].reshape(B, T, H, D).transpose(1, 2) for i in range(3))
    s = (q * (1.0 / D) ** 0.5) @ k.transpose(-1, -2)
    if key_valid is not None:
        s = s.masked_fill(~key_valid[:, None, None, :], float("-inf"))
    p = torch.softmax(s, dim=-1)
    o = (p @ v).transpose(1, 2).reshape(B, T, E)
    return F.linear(o, _p(a.out_proj.weight, dt), _p(a.out_proj.bias, dt)), p.mean(dim=1)


def _force_first(mask):
    if mask is None:
        return None
    mask = mask.clone()
    mask[:, 0] = True
    return mask


def _encoder(m, x, mask, dt):
    mask = _force_first(mask)
    for lyr in m.encoder.layers:
        sa, _ = _mha(lyr.self_attn, x, mask, dt)
        x = F.layer_norm(x + sa, lyr.norm1.normalized_shape, _p(lyr.norm1.weight, dt), _p(lyr.norm1.bias, dt),
                         lyr.norm1.eps)
        ff = F.linear(torch.relu(F.linear(x, _p(lyr.linear1.weight, dt), _p(lyr.linear1.bias, dt))),
                      _p(lyr.linear2.weight, dt), _p(lyr.linear2.bias, dt))
        x = F.layer_norm(x + ff, lyr.norm2.normalized_shape, _p(lyr.norm2.weight, dt), _p(lyr.norm2.bias, dt),
                         lyr.norm2.eps)
    if m.encoder.norm is not None:
        n = m.encoder.norm
        x = F.layer_norm(x, n.normalized_shape, _p(n.weight, dt), _p(n.bias, dt), n.eps)
    return x[:, 0, :], mask


def _lstm(m, x, mask, dt):
    r = m.lstm
    B, T, _ = x.shape
    H = r.hidden_size
    lengths = (mask.sum(1) if mask is not None else torch.full((B,), T)).clamp(1, T)
    outs = []
    for sfx in ["", "_reverse"][:2 if r.bidirectional else 1]:
        w_ih, w_hh = _p(getattr(r, "weight_ih_l0" + sfx), dt), _p(getattr(r, "weight_hh_l0" + sfx), dt)
        bias = _p(getattr(r, "bias_ih_l0" + sfx), dt) + _p(getattr(r, "bias_hh_l0" + sfx), dt)
        hs = torch.zeros(B, H, dtype=dt)
        for b in range(B):
            n = int(lengths[b])
            h = torch.zeros(H, dtype=dt)
            c = torch.zeros(H, dtype=dt)
            for s in range(n):
                t = s if sfx == "" else n - 1 - s
                z = w_ih @ x[b, t] + bias + w_hh @ h
                i, f, g, o = z[:H].sigmoid(), z[H:2 * H].sigmoid(), z[2 * H:3 * H].tanh(), z[3 * H:].sigmoid()
                c = f * c + i * g
                h = o * c.tanh()
            hs[b] = h
        outs.append(hs)
    return torch.cat(outs, dim=-1)


def _masked(m, x, mask, dt, name, weights):
    n = type(m).__name__
    if n == "MaskedSequential":
        for i, child in enumerate(m):
            cname = "%s.%d" % (name, i) if name else str(i)
            if type(child).__name__ in _MASK_MODULES and (type(child).__name__ != "LSTM" or hasattr(child, "lstm")):
                x, mask = _masked(child, x, mask, dt, cname, weights)
            else:
                x = _plain(child, x, dt)
        return x, mask
    if n == "MaskedTemporalPooling":
        return _pool(m, x, mask), mask
    if n == "LearnMaskedDefault":
        return _default(m, x, mask), mask
    if n == "TransposeMultiheadAttention":
        mask = _force_first(mask)
        y, w = _mha(m._attention, x, mask, dt)
        weights[name] = w
        return y, mask
    if n == "TransposeTransformerEncoder":
        return _encoder(m, x, mask, dt)
    if n == "LSTM":
        return _lstm(m, x, mask, dt), mask
    raise NotImplementedError(n)


def _plain(m, x, dt):
    n = type(m).__name__
    if n in ("Dropout", "Identity"):
        return x
    if n == "LayerNorm":
        return F.layer_norm(x, m.normalized_shape, _p(m.weight, dt), _p(m.bias, dt), m.eps)
    if n == "Linear":
        return F.linear(x, _p(m.weight, dt), _p(m.bias, dt))
    if n == "PositionalEncoding":
        return x + _p(m.pe, dt)[:, :x.size(1), :]
    raise NotImplementedError(n)


def _fuse(m, xs):
    n = type(m).__name__
    if n == "ConcatFusion":
        return torch.cat(xs, dim=-1)
    if n == "TemporalConcatFusion":
        return torch.cat(xs, dim=1)
    if n == "ReduceFusion":
        return m.reduce_fn(torch.stack(xs))
    raise NotImplementedError(n)


def masked_forward(m, x, mask=None, dtype=torch.float32):
    """The forward of a case's root module (testing.masked_call's convention; every stream of a MaskedMultiPathWay
    takes ``x`` and ``mask``)."""
    weights = {}
    x = x.detach().cpu().to(dtype)
    mask = None if mask is None else mask.detach().cpu()
    n = type(m).__name__
    with torch.no_grad():
        if n == "MaskedMultiPathWay":
            outs = []
            for i, blk in enumerate(m.multipathway_blocks):
                outs.append(_masked(blk, x, mask, dtype, "multipathway_blocks.%d" % i, weights)[0])
            y = _fuse(m.multipathway_fusion, outs)
        elif n == "PositionalEncoding":
            y = _plain(m, x, dtype)
        else:
            y = _masked(m, x, mask, dtype, "", weights)[0]
    return y, weights
