"""In-place weight refresh of a compiled plan (pv_weights_refresh), for BYOL's momentum backbone.

A plan's constants are derived from the module's parameters once, on the host, when it is built (packing.py).  After
the module's fp32 parameters change IN PLACE (pv_ema_update), ``WeightsRefresh`` re-derives every such constant on the
device, into the same buffers, so the plan's captured CUDA graph stays valid and no compile runs.

When the refresh is built, each constant is classified:
- a BatchNorm fold vector (packing.fold_bn, recognised by the origin it records): refreshed by the fp64 fold on the
  device from the module's current parameters and running statistics;
- a pure re-layout of ONE parameter (packed weights, zero padding included): a gather map, packed element <- source
  element or zero, found by lowering the same module again with its parameters replaced by index codes and reading the
  codes back out of the packed constants.  Codes are integers of at most 2048 (exact in f16): the parameter number in
  two passes (k + 1 and 2 (k + 1): an element that does not scale is not parameter data), and the element index in
  base-1024 digits, one pass per digit;
- independent of the parameters (identical in the two parameter-number passes): left as it is.
Anything else (a constant mixing parameters, or computed from them other than by re-layout or the BatchNorm fold, such
as the BatchNorm MViT's W diag(s) folded into f16 weights) makes the plan non-refreshable: ``build`` returns None and
the caller compiles again.  The tables are checked once before use: a refresh right after the compile must rewrite
every constant with its own bytes.
"""
import copy
import struct

import torch

from .. import _lib as L

CHUNK = 4096            # elements per block of pv_weights_refresh (csrc/pv_contrastive.cu REFRESH_CHUNK)
_BASE = 1024


def _lower_consts(model, shapes, dtype, extra):
    from .lower import lower_only
    plan, _ = lower_only(model, [torch.empty(s) for s in shapes] if len(shapes) > 1 else torch.empty(shapes[0]),
                         dtype, extra)
    return [t.double() for t in plan.consts], plan.const_folds


class WeightsRefresh:
    def __init__(self, cm, params, gather, folds):
        dev = cm.plan.device
        self.cm = cm
        self.params = params
        self.ptrs = [p.data_ptr() for p in params]
        jobs, chunks, maps, off = [], [], [], 0
        for j, (t, slot, m) in enumerate(gather):
            jobs += [t.data_ptr(), L.PV_F16 if t.dtype == torch.float16 else L.PV_F32, t.numel(), off, slot]
            chunks += [(j << 40) | c for c in range(0, t.numel(), CHUNK)]
            maps.append(m)
            off += m.numel()
        self.n_chunks = len(chunks)
        self.jobs = torch.tensor(jobs or [0], dtype=torch.int64).to(dev)
        self.chunks = torch.tensor(chunks or [0], dtype=torch.int64).to(dev)
        self.map = (torch.cat(maps) if maps else torch.zeros(1, dtype=torch.int32)).to(dev)
        self.srcs = torch.tensor(self.ptrs or [0], dtype=torch.int64).to(dev)
        fj = []
        for sd, bd, c_out, srcs, eps in folds:
            fj += [sd.data_ptr(), bd.data_ptr(), c_out] + [0 if s is None else s.data_ptr() for s in srcs]
            fj.append(struct.unpack("<q", struct.pack("<d", float(eps)))[0])
        self.n_folds = len(folds)
        self.folds = torch.tensor(fj or [0], dtype=torch.int64).to(dev)
        self.device = dev

    @classmethod
    def build(cls, cm, model, example_inputs, dtype, extra=()):
        """The refresh of the compiled plan ``cm`` of ``model``, or None when the plan is not refreshable."""
        ins = list(example_inputs) if isinstance(example_inputs, (list, tuple)) else [example_inputs]
        shapes = [tuple(t.shape) for t in ins]
        consts, origins = cm.plan.consts, cm.plan.const_folds
        params = list(model.parameters())
        if len(params) > 2047 or any(p.dtype != torch.float32 or p.device != cm.plan.device or not p.is_contiguous()
                                     for p in params):
            return None
        owned = {id(t) for t in list(model.parameters()) + list(model.buffers())}
        work = copy.deepcopy(model).cpu()
        wparams = list(work.parameters())
        digits = 1
        while max([p.numel() for p in params] + [1]) > _BASE ** digits:
            digits += 1

        def encoded(fill):
            with torch.no_grad():
                for k, p in enumerate(wparams):
                    p.copy_(fill(k, p))
            return _lower_consts(work, shapes, dtype, extra)

        a, fa = encoded(lambda k, p: torch.full(p.shape, float(k + 1)))
        b, _ = encoded(lambda k, p: torch.full(p.shape, float(2 * (k + 1))))
        ds = [encoded(lambda k, p, d=d: ((torch.arange(p.numel()) // _BASE ** d) % _BASE + 1).float().reshape(p.shape))[0]
              for d in range(digits)]
        if len(a) != len(consts) or [o is None for o in fa] != [o is None for o in origins]:
            return None
        gather, folds, pending = [], [], {}
        for j, t in enumerate(consts):
            o = origins[j]
            if o is not None:
                conv_bias, bn, c_out, which = o
                srcs = [conv_bias] + ([None] * 4 if bn is None else
                                      [bn.weight, bn.bias, bn.running_mean, bn.running_var])
                if all(s is None for s in srcs):
                    continue                                      # ones / zeros: independent of the parameters
                if any(s is not None and id(s) not in owned for s in srcs) or (bn is not None and bn.running_var is None):
                    return None
                key = (id(conv_bias), id(bn), c_out)
                if which == 0:
                    pending[key] = t
                elif key in pending:
                    folds.append((pending.pop(key), t, c_out, srcs, 0.0 if bn is None else bn.eps))
                else:
                    return None
                continue
            if t.dtype not in (torch.float16, torch.float32) or a[j].shape != t.shape:
                return None
            aj, bj = a[j].reshape(-1), b[j].reshape(-1)
            if torch.equal(aj, bj):
                continue                                          # independent of the parameters
            data = bj != aj
            if not (torch.equal(bj[data], 2 * aj[data]) and bool((aj[~data] == 0).all())):
                return None
            slots = torch.unique(aj[data])
            if slots.numel() != 1:
                return None                                       # mixes parameters
            slot = int(slots[0]) - 1
            if slots[0] != slot + 1 or not 0 <= slot < len(params):
                return None
            idx = torch.zeros(aj.numel(), dtype=torch.float64)
            for d in range(digits):
                dig = ds[d][j].reshape(-1)[data]
                if not bool(((dig >= 1) & (dig <= _BASE) & (dig == dig.round())).all()):
                    return None
                idx[data] += (dig - 1) * float(_BASE ** d)
            if bool((idx[data] >= params[slot].numel()).any()):
                return None
            m = torch.full((aj.numel(),), -1, dtype=torch.int32)
            m[data] = idx[data].to(torch.int32)
            gather.append((t, slot, m))
        if pending:
            return None
        r = cls(cm, params, gather, folds)
        before = [t.clone() for t in consts]
        r()
        torch.cuda.synchronize(cm.plan.device)
        if not all(torch.equal(x.view(torch.uint8) if x.dtype != torch.uint8 else x,
                               y.view(torch.uint8) if y.dtype != torch.uint8 else y) for x, y in zip(before, consts)):
            for x, y in zip(before, consts):
                y.copy_(x)
            return None
        return r

    def __call__(self):
        """Rewrite the plan's parameter-derived constants from the module's current parameters (one call, two
        launches, on the current stream)."""
        if [p.data_ptr() for p in self.params] != self.ptrs:
            raise RuntimeError("a parameter of the refreshable plan moved; compile the plan again")
        L.check(L.load().pv_weights_refresh(self.jobs.data_ptr(), self.chunks.data_ptr(), self.n_chunks,
                                            self.map.data_ptr(), self.srcs.data_ptr(), self.folds.data_ptr(),
                                            self.n_folds, torch.cuda.current_stream(self.device).cuda_stream),
                "pv_weights_refresh")

