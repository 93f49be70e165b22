"""Static execution plan: symbolic NDHWC tensors + a list of libpvb200 launches.

A ``TRef`` is a channels-last-3d activation living in a (possibly shared) buffer:
element (n,t,h,w,c) is at ``buf + ((n*T+t)*H+h)*W+w) * row_stride + ch_off + c``.  Because ops
resolve pointers only when they run, a tensor can be *retargeted* into a channel slice of a wider
buffer after it was produced - that is how ``torch.cat([slow, fuse], dim=1)``
(reference models/slowfast.py:728) disappears: both producers write straight into the concat
buffer.
"""
import ctypes as C

import torch

from .. import _lib as L
from . import packing as PK

_TORCH_DT = {L.PV_F16: torch.float16, L.PV_F32: torch.float32, L.PV_U8: torch.uint8}
_ESIZE = {L.PV_F16: 2, L.PV_F32: 4, L.PV_U8: 1}
# SM count of the H100 SXM: routing thresholds that count waves of work.  Lowering runs without a device, so the plan
# (and the goldens that pin it) must not depend on the GPU it is built on.
H100_SXM_SMS = 132


class Buf:
    def __init__(self, numel, dt):
        self.numel = int(numel)
        self.dt = dt
        self.tensor = None


class RawIn:
    """Plan input passed through untouched (see Plan.raw_input)."""

    def __init__(self, tensor):
        self.tensor = tensor


class MaskRef:
    """A (B, T) u8 mask of a plan (non-zero = valid step): the staged plan input (``tensor``) or a plan buffer."""

    def __init__(self, B, T, tensor=None, buf=None):
        self.B, self.T = int(B), int(T)
        self.tensor, self.buf = tensor, buf

    def ptr(self):
        return (self.tensor if self.tensor is not None else self.buf.tensor).data_ptr()

    def io(self):
        return (self.buf,) if self.buf is not None else ()


class TRef:
    def __init__(self, buf, N, T, H, W, C, Cp=None, ch_off=0, row_stride=None):
        self.buf = buf
        self.N, self.T, self.H, self.W = int(N), int(T), int(H), int(W)
        self.C = int(C)
        self.Cp = PK.pad8(C) if Cp is None else int(Cp)
        self.ch_off = int(ch_off)
        self.row_stride = self.Cp if row_stride is None else int(row_stride)
        self.lazy_src = None      # network input whose NCDHW->NDHWC conversion is emitted by its first consumer
        self.padw = None          # (w_pad, w_phys): rows physically zero-padded along W (window-mode stems)

    @property
    def npos(self):
        return self.T * self.H * self.W

    @property
    def dt(self):
        return self.buf.dt

    def ptr(self):
        return self.buf.tensor.data_ptr() + self.ch_off * _ESIZE[self.buf.dt]

    def retarget(self, buf, ch_off, row_stride):
        self.buf, self.ch_off, self.row_stride = buf, int(ch_off), int(row_stride)

    def shape5(self):
        return (self.N, self.C, self.T, self.H, self.W)

    def __repr__(self):
        return "TRef(N=%d,C=%d(%d),T=%d,H=%d,W=%d,off=%d,rs=%d)" % (
            self.N, self.C, self.Cp, self.T, self.H, self.W, self.ch_off, self.row_stride)


def _may_overlap(a, b):
    """False only when two plan items of one buffer provably touch different elements: TRefs over the same rows whose
    channel slices [ch_off, ch_off + Cp) do not meet (the parts of a concat buffer)."""
    if not (isinstance(a, TRef) and isinstance(b, TRef)) or a.padw is not None or b.padw is not None:
        return True
    if a.row_stride != b.row_stride or a.N * a.npos != b.N * b.npos:
        return True
    return a.ch_off < b.ch_off + b.Cp and b.ch_off < a.ch_off + a.Cp


def _conv_out(i, k, s, p, d):
    return (i + 2 * p - d * (k - 1) - 1) // s + 1


class Plan:
    """Collects launches; ``finalize`` allocates, ``run`` replays (eagerly or as a CUDA graph)."""

    def __init__(self, device, dt=L.PV_F16):
        self.lib = L.load()
        self.device = torch.device(device)
        self.dt = dt
        self.ops = []          # (name, closure(stream_ptr))
        self.meta = []         # per-op {name, kind, flops, bytes} (algorithmic figures for the roofline)
        # per op: what it computes, in torch terms ({"kind": "conv", "x": TRef, "weight": ..., "y": TRef, ...}), or None
        # for an op that produces no value of its own (the SE-sum clear).  Tensors are TRefs, resolved when read, since
        # concat_channels retargets them after their producer was emitted.  Kept out of meta, which is dumped as JSON.
        self.op_spec = []
        self.attention_calls = []   # per attention op: its problem (B, H, Nq, Nk, D, scale, normalize, residual)
        self.side_outputs = []      # (weakref to module, Buf, shape): per-module results besides the output (attention weights)
        self.bufs = []
        self.consts = []       # keep device parameter tensors alive
        self.const_folds = []  # per const: (conv_bias, bn, c_out, 0 scale | 1 bias) of a packing.fold_bn vector, else None
        self.zero_bufs = []    # f32 accumulators that must be cleared every run (SE sums)
        self.finalized = False
        self.graph = None
        self.stats = {"tcgen05": 0, "direct": 0, "depthwise": 0, "other": 0}
        # ---- lanes: independent branches of the network (SlowFast pathways) run on separate CUDA streams /
        #      graph branches.  Every op records the tensors it reads / writes; finalize() turns cross-lane
        #      read-after-write, write-after-read and write-after-write pairs into event waits (see _schedule).
        self.lane = 0          # lane of the ops being emitted (set by the lowering)
        self.op_lane = []
        self.op_io = []        # (reads, writes) as lists of TRef / Buf, or None = unknown (acts as a full barrier)
        self.sched = None
        # f16 engine, MViT: the residual token stream (16 blocks x 2 adds) is kept in fp32 - branch outputs stay f16, the
        # add + LayerNorm is one kernel (pv_add_layernorm).
        self.trunk32 = dt == L.PV_F16
        self._streams = {}
        self._events = {}

    # ---- memory --------------------------------------------------------------------------
    def new_buf(self, numel, dt=None):
        b = Buf(numel, self.dt if dt is None else dt)
        self.bufs.append(b)
        return b

    def new_tensor(self, N, T, H, W, C, Cp=None, dt=None):
        Cp = PK.pad8(C) if Cp is None else Cp
        b = self.new_buf(N * T * H * W * Cp, dt)
        return TRef(b, N, T, H, W, C, Cp)

    def const(self, t, dtype=None):
        fold = getattr(t, "_pv_fold", None)
        t = t.detach().to(device=self.device, dtype=dtype if dtype is not None else t.dtype).contiguous()
        self.consts.append(t)
        self.const_folds.append(fold if dtype is None else None)   # packing.fold_bn origin (engine/refresh.py)
        return t

    def finalize(self):
        for b in self.bufs:
            if b.tensor is None:
                # zero-init so that pad lanes / never-written slices are finite
                b.tensor = torch.zeros(max(b.numel, 8), dtype=_TORCH_DT[b.dt], device=self.device)
        self._schedule()
        self.finalized = True

    def _schedule(self):
        """Cross-lane dependencies.  For op i on lane L: for every other lane M, the LAST op j < i on M that i
        conflicts with (stream order covers the earlier ones): j wrote a buffer i reads (read-after-write), or i
        writes elements j read or wrote (write-after-read, write-after-write: in-place ops such as the SE scale and
        the activations, the SE-sum accumulators).  Writes are compared by element footprint (_may_overlap), so two
        lanes writing disjoint channel slices of one concat buffer stay concurrent.  Ops with unknown I/O are full
        barriers."""
        def items_of(items):
            out = []
            for t in items or ():
                b = t if isinstance(t, Buf) else getattr(t, "buf", None)
                if b is not None:
                    out.append((b, t))
            return out
        n = len(self.ops)
        lanes = sorted(set(self.op_lane)) if self.op_lane else [0]
        waits = [[] for _ in range(n)]      # op -> list of op indices (on other lanes) to wait for
        writers = {}                        # id(buf) -> {lane: last writer op}
        touched = {}                        # id(buf) -> {lane: [(op, item)]} every read and write, in program order
        last_on_lane = {}
        last_barrier = None                 # last op with unknown I/O
        waited = {}                         # lane -> {other lane: latest op already waited for}
        for i in range(n):
            L = self.op_lane[i]
            io = self.op_io[i]
            need = {}
            if io is None:
                for M, j in last_on_lane.items():
                    if M != L:
                        need[M] = j
            else:
                for b, _ in items_of(io[0]):
                    for M, j in writers.get(id(b), {}).items():
                        if M != L:
                            need[M] = max(need.get(M, -1), j)
                for b, t in items_of(io[1]):
                    for M, acc in touched.get(id(b), {}).items():
                        if M != L:
                            j = next((j for j, u in reversed(acc) if _may_overlap(t, u)), -1)
                            need[M] = max(need.get(M, -1), j)
                if last_barrier is not None and self.op_lane[last_barrier] != L:
                    M = self.op_lane[last_barrier]
                    need[M] = max(need.get(M, -1), last_barrier)
            # a lane never needs to wait twice for the same (or an earlier) op of another lane
            seen = waited.setdefault(L, {})
            keep = []
            for M, j in sorted(need.items()):
                if seen.get(M, -1) < j:
                    seen[M] = j
                    keep.append(j)
            waits[i] = sorted(keep)
            if io is None:
                last_barrier = i
            else:
                for b, t in items_of(io[0]) + items_of(io[1]):
                    touched.setdefault(id(b), {}).setdefault(L, []).append((i, t))
                for b, _ in items_of(io[1]):
                    writers.setdefault(id(b), {})[L] = i
            last_on_lane[L] = i
        signals = sorted(set(j for w in waits for j in w))
        self.sched = {"lanes": lanes, "waits": waits, "signals": set(signals), "last_on_lane": last_on_lane}

    def bytes_allocated(self):
        return sum(b.numel * _ESIZE[b.dt] for b in self.bufs)

    # ---- execution -----------------------------------------------------------------------
    def add(self, name, fn, kind="other", flops=0.0, nbytes=0.0, reads=None, writes=None, spec=None):
        """reads / writes: the TRefs (or Bufs) the launch touches; leave both None for "unknown" (the op then
        orders against everything on the other lanes).  spec: the op_spec record of the launch."""
        self.ops.append((name, fn))
        self.op_spec.append(spec)
        self.meta.append({"name": name, "kind": kind, "flops": float(flops), "bytes": float(nbytes), "lane": self.lane})
        self.stats[kind] = self.stats.get(kind, 0) + 1
        self.op_lane.append(self.lane)
        self.op_io.append(None if reads is None and writes is None else (list(reads or ()), list(writes or ())))

    def profile(self, iters=3):
        """Per-launch device times (ms, mean over `iters`) measured with CUDA events on the
        launching stream (torch's current stream); eager replay, one event pair per launch."""
        assert self.finalized
        stream = torch.cuda.current_stream(self.device)
        sp = stream.cuda_stream
        n = len(self.ops)
        acc = [0.0] * n
        for it in range(iters + 1):
            evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
            for (e0, e1), (_, fn) in zip(evs, self.ops):      # single stream: lanes are ignored here
                e0.record(stream)
                fn(sp)
                e1.record(stream)
            stream.synchronize()
            if it == 0:
                continue   # warm-up pass
            for i, (e0, e1) in enumerate(evs):
                acc[i] += e0.elapsed_time(e1)
        return [a / iters for a in acc]

    def run(self, stream_ptr, single_stream=False):
        """Enqueue every launch.  With more than one lane the extra lanes run on side streams that fork from /
        join back into ``stream_ptr`` with events, so a CUDA-graph capture of this call records a graph with
        parallel branches (and an eager call overlaps them the same way)."""
        assert self.finalized
        lanes = self.sched["lanes"]
        if single_stream or len(lanes) <= 1:
            for _, fn in self.ops:
                fn(stream_ptr)
            return
        main = torch.cuda.ExternalStream(stream_ptr, device=self.device)
        streams = {lanes[0]: main}
        for L in lanes[1:]:
            if L not in self._streams:
                self._streams[L] = torch.cuda.Stream(device=self.device)
            streams[L] = self._streams[L]
        ev = self._events

        def event(key):
            e = ev.get(key)
            if e is None:
                e = ev[key] = torch.cuda.Event()
            return e
        fork = event("fork")
        fork.record(main)
        for L in lanes[1:]:
            streams[L].wait_event(fork)
        waits, signals = self.sched["waits"], self.sched["signals"]
        for i, (_, fn) in enumerate(self.ops):
            st = streams[self.op_lane[i]]
            for j in waits[i]:
                st.wait_event(event(j))
            fn(st.cuda_stream)
            if i in signals:
                event(i).record(st)
        for L in lanes[1:]:
            e = event(("join", L))
            e.record(streams[L])
            main.wait_event(e)

    def num_launches(self):
        return len(self.ops)

    # =====================================================================================
    # op emitters
    # =====================================================================================
    def emit_input_ncdhw(self, static_in, C, c_pad):
        """static_in: torch tensor [N,C,T,H,W] (f32|f16) whose storage is fixed for the plan.
        The layout conversion is emitted lazily by the first consumer (a stem conv may ask for
        physically W-padded rows, see pv_igemm.cu window mode)."""
        N, Cc, T, H, W = static_in.shape
        assert Cc == C
        out = TRef(None, N, T, H, W, C, Cp=c_pad)
        out.lazy_src = static_in
        return out

    def materialize_input(self, x, w_pad=0, w_phys=0):
        if x.lazy_src is None:
            return x
        src = x.lazy_src
        x.lazy_src = None
        N, C, T, H, W = src.shape
        src_dt = L.PV_F32 if src.dtype == torch.float32 else L.PV_F16
        lib = self.lib
        if w_pad > 0:
            x.buf = self.new_buf(N * T * H * w_phys * x.Cp + 64 * x.Cp)
            x.padw = (w_pad, w_phys)

            def fn(stream):
                L.check(lib.pv_ncdhw_to_ndhwc_padw(src.data_ptr(), src_dt, x.ptr(), x.dt, N, C, T, H, W, x.Cp,
                                                  w_pad, w_phys, stream), "pv_ncdhw_to_ndhwc_padw")
            self.add("ncdhw_to_ndhwc_padw", fn, "other", 0.0, src.numel() * src.element_size() + N * T * H * w_phys * x.Cp * 2,
                     reads=(), writes=(x,), spec={"kind": "to_ndhwc", "src": src, "y": x})
        else:
            x.buf = self.new_buf(N * T * H * W * x.Cp)

            def fn(stream):
                L.check(lib.pv_ncdhw_to_ndhwc(src.data_ptr(), src_dt, x.ptr(), x.dt, N, C, T, H, W, x.Cp,
                                              x.row_stride, stream), "pv_ncdhw_to_ndhwc")
            self.add("ncdhw_to_ndhwc", fn, "other", 0.0, src.numel() * src.element_size() + N * T * H * W * x.Cp * 2,
                     reads=(), writes=(x,), spec={"kind": "to_ndhwc", "src": src, "y": x})
        return x

    def emit_conv(self, x, weight, conv_bias, bn, stride, padding, dilation, groups, act=L.ACT_NONE,
                  residual=None, name="conv", force_algo=None, se_sums=False, addend=None, folded=None):
        """Conv3d (+folded BN/bias) (+residual) (+activation) (+addend).  weight: [Co, Ci/g, kt, kh, kw].
        se_sums (depthwise only): also accumulate the per-(sample, channel) sums of the output inside
        the conv kernel (Squeeze-Excitation statistics); the buffer is attached as ``y.se_sums``.
        addend: (a, c_off) - a (N, T' in {To, 1}, 1, 1, C) tensor added after the activation, output channel c taking
        a's channel c_off + c (pv_conv3d_desc.addend).  folded: precomputed (scale, bias) of length Co instead of
        conv_bias / bn."""
        co, cig, kt, kh, kw = weight.shape
        ci = cig * groups
        if ci != x.C:
            # same error type the reference raises for a wrong channel count
            raise RuntimeError("conv %s expects %d input channels, got %d" % (name, ci, x.C))
        st, sh, sw = stride
        pt, ph, pw = padding
        dlt, dlh, dlw = dilation
        To, Ho, Wo = _conv_out(x.T, kt, st, pt, dlt), _conv_out(x.H, kh, sh, ph, dlh), _conv_out(x.W, kw, sw, pw, dlw)
        if min(To, Ho, Wo) <= 0:
            raise RuntimeError("conv %s: kernel larger than (padded) input" % name)
        co_pad = PK.pad8(co)
        if addend is not None:
            a, a_off = addend
            # torch broadcasting of a (N, C, T', 1, 1) tensor against the (N, C, To, Ho, Wo) output
            if a.N != x.N or a.H != 1 or a.W != 1 or a.T not in (To, 1):
                raise RuntimeError("conv %s: addend of shape %s does not broadcast to the output %s" % (
                    name, a.shape5(), (x.N, co, To, Ho, Wo)))
            if a_off + co_pad > a.Cp:
                raise RuntimeError("conv %s: addend has %d channels, the output needs %d from channel %d" % (
                    name, a.C, co, a_off))
        depthwise = groups != 1 and groups == ci == co
        if depthwise and addend is not None:
            raise NotImplementedError("conv %s: depthwise convolutions take no addend" % name)
        span = None
        if groups != 1 and not depthwise:
            # grouped conv (ResNeXt-style group counts, CSN with several channels per group): the grouped mode of the
            # TMA-fed kernel when the library takes the shape, else the dense convolution with block-diagonal weights
            # (one group span, C % 8 != 0, non-square groups, f32, forced CUDA-core algorithm)
            if self.dt == L.PV_F16 and force_algo in (None, L.ALGO_TCGEN05) and x.Cp == ci and co_pad == co:
                probe = self._conv_desc(x, (To, Ho, Wo), co_pad, (kt, kh, kw), stride, padding, dilation, groups, act,
                                        residual, co_pad, 0)
                if addend is not None:
                    probe.addend, probe.add_n_stride = 256, a.T * a.row_stride      # layout probe, see below
                    probe.add_t_stride, probe.add_ch_off = (a.row_stride if a.T == To > 1 else 0), a_off
                taken, span_g, span_k, _ = L.group_span(probe)
                span = (span_g, span_k) if taken else None
            if span is None:
                return self.emit_conv(x, PK.expand_grouped_dense(weight, groups), conv_bias, bn, stride, padding,
                                      dilation, 1, act, residual, name, force_algo=force_algo, se_sums=se_sums,
                                      addend=addend, folded=folded)
        if residual is not None:
            self.materialize_input(residual)
        esz = _ESIZE[self.dt]
        m_out = x.N * To * Ho * Wo
        flops = 2.0 * m_out * co * cig * kt * kh * kw
        nbytes = (x.N * x.npos * ci + m_out * co * (2 if residual is not None else 1)) * esz + weight.numel() * esz
        stem_candidate = (x.lazy_src is not None and self.dt == L.PV_F16 and force_algo in (None, L.ALGO_TCGEN05)
                          and groups == 1 and x.Cp == 4 and kt > 1 and residual is None and addend is None and dlw == 1
                          and pw > 0)
        # Narrow stems with a temporal extent run as two launches, `.taps` (the convolution's tensor-core pass) and
        # `.tapsum` (pv_temporal_tap_sum: folded BN, activation), on one of two routes:
        # ---- at least one full wave of output rows: the streaming stem (csrc/pv_stem_stream.cu) walks every output
        #      row over all input frames and sums the kt temporal taps in fp32 registers, so `.taps` writes the Co
        #      channels of the pre-BN sum once (rounded to f16 once); `.tapsum` is then the BN / activation pass over
        #      it (one tap).  With fewer rows than SMs the factored route fills the machine better (its taps pass has
        #      kt times more tiles).
        if stem_candidate and x.N * Ho * -(-Wo // 128) >= H100_SXM_SMS:
            wp, w_phys, lead, win = self._stem_window(x, kw, sw, pw, Wo)
            d = self._conv_desc(x, (To, Ho, Wo), co_pad, (kt, kh, kw), stride, padding, dilation, 1, L.ACT_NONE, None,
                                co_pad, win)
            d.x_w_pad, d.x_w_phys = wp, w_phys
            if self.lib.pv_conv3d_stem_stream_supported(C.byref(d)):
                ysum = self._emit_stem_stream(x, d, weight, co, lead, name + ".taps", flops, nbytes)
                return self._emit_tap_sum(ysum, To, To, co, 1, 1, 0, 1, conv_bias, bn, act, name)
        # ---- factor (kt,kh,kw) -> (1,kh,kw) with kt*Co channels (all temporal taps in one tensor-core pass, each
        #      tap's partial rounded to f16 and written out) + the temporal tap sum.  Only below 16 output channels:
        #      from there the direct convolution is already a full wgmma width and writes no kt-fold intermediate
        #      (CSN's 3x7x7 3->64 stem at batch 8: 0.96 ms direct, 2.10 ms factored, DESIGN.md).
        if stem_candidate and co_pad < 16 and co_pad * kt <= 256 and (sw * x.Cp * 2) % 16 == 0 and kw * x.Cp <= 64 and sh <= 8:
            w2 = torch.zeros(kt * co_pad, cig, 1, kh, kw, dtype=weight.dtype)
            wsrc = weight.detach().cpu()
            for j in range(kt):
                w2[j * co_pad: j * co_pad + co] = wsrc[:, :, j:j + 1]
            yk = self.emit_conv(x, w2, None, None, (1, sh, sw), (0, ph, pw), (1, dlh, dlw), 1, L.ACT_NONE, None,
                                name + ".taps")
            return self._emit_tap_sum(yk, x.T, To, co, kt, st, pt, dlt, conv_bias, bn, act, name)
        # ---- network input: pick the layout its first consumer wants
        window = False
        if x.lazy_src is not None:
            window = (self.dt == L.PV_F16 and force_algo in (None, L.ALGO_TCGEN05) and groups == 1 and x.Cp == 4
                      and dlw == 1 and (sw * x.Cp * 2) % 16 == 0 and (kw + 1) * x.Cp <= 64 and kt * kh <= 64
                      and st * sh <= 8 and pw > 0)
            if window:
                wp, w_phys, _, _ = self._stem_window(x, kw, sw, pw, Wo)
                self.materialize_input(x, w_pad=wp, w_phys=w_phys)
            else:
                self.materialize_input(x)
        elif x.padw is not None:
            raise RuntimeError("W-padded stem input can only feed one window-mode convolution")
        y = self.new_tensor(x.N, To, Ho, Wo, co, Cp=co_pad)
        if folded is None:
            scale, bias = PK.fold_bn(conv_bias, bn, co, co_pad)
        else:
            scale, bias = (torch.cat([t.float(), torch.zeros(co_pad - co)]) for t in folded)
        scale_d, bias_d = self.const(scale), self.const(bias)
        tdt = _TORCH_DT[self.dt]
        ci_pad = x.Cp
        ci_pad64 = ci_pad if ci_pad < 64 else PK.pad_to(ci_pad, 64)   # < 64: gather-fed kernel, un-padded taps
        if span is not None:
            ci_pad64 = span[1]                                          # grouped mode: weights packed at the span width

        d = self._conv_desc(x, (To, Ho, Wo), co_pad, (kt, kh, kw), stride, padding, dilation,
                            ci_pad if depthwise else (groups if span is not None else 1), act, residual, y.row_stride,
                            ci_pad64)
        if addend is not None:
            d.add_n_stride = a.T * a.row_stride
            d.add_t_stride = a.row_stride if a.T == To > 1 else 0
            d.add_ch_off = a_off
            # the buffer is allocated at finalize(): until then an aligned placeholder, so that the routing probes
            # below check the addend's layout rules as the launch will (a.ptr() is 16-byte aligned: own buffer)
            d.addend = 256

            def set_addend():
                d.addend = a.ptr()
        else:
            def set_addend():
                pass
        if window:
            d.x_w_pad, d.x_w_phys = x.padw
            w_lead = PK.window_lead(x.padw[0], pw, x.Cp)
            d.ci_pad64 = PK.window_elems(kw, x.Cp, w_lead)

        stem_rows, zero_row = False, None
        if depthwise:
            algo, kind = L.ALGO_DIRECT, "depthwise"
            w_d = self.const(PK.pack_depthwise(weight, co_pad, tdt))
        elif span is not None:
            algo, kind = L.ALGO_TCGEN05, "grouped"
            w_d = self.const(PK.pack_grouped_tcgen05(weight, groups, span[0], span[1]))
        else:
            want_tc = self.dt == L.PV_F16 and bool(self.lib.pv_conv3d_tcgen05_supported(C.byref(d)))
            if force_algo is not None:
                want_tc = force_algo == L.ALGO_TCGEN05
            if window and not want_tc:
                raise RuntimeError("internal: window-mode stem rejected by the library: " + L.last_error())
            stem_rows = window and want_tc and residual is None and bool(self.lib.pv_conv3d_stem_rows_supported(C.byref(d)))
            if stem_rows:
                # zero-copy im2col over raw input rows (csrc/pv_stem.cu): its own weight layout and entry point
                algo, kind = L.ALGO_TCGEN05, "tcgen05"
                w_d = self.const(PK.pack_stem_rows(weight, x.Cp, co_pad, w_lead))
                zero_row = self.const(torch.zeros(4096, dtype=torch.float16))
            elif want_tc:
                algo, kind = L.ALGO_TCGEN05, "tcgen05"
                w_d = self.const(PK.pack_dense_window(weight, x.Cp, co_pad, w_lead) if window
                                 else PK.pack_dense_tcgen05(weight, ci_pad64, co_pad))
            else:
                algo, kind = L.ALGO_DIRECT, "direct"
                w_d = self.const(PK.pack_dense_direct(weight, ci_pad, co_pad, tdt))
        lib = self.lib
        sums = None
        if se_sums and depthwise and residual is None and act == L.ACT_NONE:
            sums = self.new_buf(2 * x.N * co_pad, L.PV_F32)     # one int64 (fixed point) per (sample, channel)
            self.zero_bufs.append(sums)
            y.se_sums = sums

            def fn_zero(stream):
                L.check(lib.pv_zero_f32(sums.tensor.data_ptr(), 2 * x.N * co_pad, stream), "pv_zero_f32")
            self.add(name + ".se_zero", fn_zero, reads=(), writes=(sums,))

        def fn_dw(stream):
            d.x_row_stride, d.y_row_stride = x.row_stride, y.row_stride
            L.check(lib.pv_dwconv3d_fwd(C.byref(d), x.ptr(), w_d.data_ptr(), scale_d.data_ptr(), bias_d.data_ptr(),
                                        y.ptr(), sums.tensor.data_ptr() if sums is not None else None, stream),
                    "pv_dwconv3d_fwd(%s)" % name)

        def fn_stem(stream):
            d.x_row_stride, d.y_row_stride = x.row_stride, y.row_stride
            set_addend()
            L.check(lib.pv_conv3d_stem_rows_fwd(C.byref(d), x.ptr(), w_d.data_ptr(), scale_d.data_ptr(), bias_d.data_ptr(),
                                                zero_row.data_ptr(), y.ptr(), stream), "pv_conv3d_stem_rows_fwd(%s)" % name)

        def fn(stream):
            d.x_row_stride, d.y_row_stride = x.row_stride, y.row_stride   # may have been retargeted
            d.res_row_stride = residual.row_stride if residual is not None else 0
            set_addend()
            L.check(lib.pv_conv3d_fwd(C.byref(d), algo, x.ptr(), w_d.data_ptr(), scale_d.data_ptr(),
                                      bias_d.data_ptr(), residual.ptr() if residual is not None else None,
                                      y.ptr(), stream), "pv_conv3d_fwd(%s)" % name)
        if stem_rows:
            self.stats["stem_rows"] = self.stats.get("stem_rows", 0) + 1
        spec = {"kind": "conv", "route": kind, "x": x, "weight": weight, "scale": scale[:co], "bias": bias[:co],
                "stride": tuple(stride), "padding": tuple(padding), "dilation": tuple(dilation), "groups": groups,
                "act": act, "residual": residual, "addend": addend, "y": y, "se_sums": sums}
        self.add(name, fn_stem if stem_rows else (fn_dw if (depthwise and residual is None) else fn), kind, flops, nbytes,
                 reads=(x,) + ((residual,) if residual is not None else ()) + ((a,) if addend is not None else ())
                 + ((sums,) if sums is not None else ()),          # the SE sums accumulate onto the cleared buffer
                 writes=(y,) + ((sums,) if sums is not None else ()), spec=spec)
        if addend is not None:
            self.meta[-1]["addend"] = (a.buf, a_off)
        return y

    @staticmethod
    def _stem_window(x, kw, sw, pw, Wo):
        """(w_pad, w_phys, lead, window elements) of the physically W-padded network input a window-mode stem reads;
        the left pad is rounded up to 4 pixels, which enables the 4-pixel conversion kernel."""
        wp = (pw + 3) // 4 * 4
        lead = PK.window_lead(wp, pw, x.Cp)
        win = PK.window_elems(kw, x.Cp, lead)
        need = wp - pw + max(x.W + 2 * pw, (Wo - 1) * sw + (win + x.Cp - 1) // x.Cp)
        return wp, (need + 3) // 4 * 4, lead, win

    def _emit_tap_sum(self, yk, Ti, To, co, kt, st, pt, dlt, conv_bias, bn, act, name):
        """``name``.tapsum: y = act(scale * sum over the kt channel groups of yk at frames t*st + j*dlt - pt + bias)
        with the folded BN of the convolution (pv_temporal_tap_sum)."""
        co_pad = PK.pad8(co)
        y = self.new_tensor(yk.N, To, yk.H, yk.W, co, Cp=co_pad)
        scale, bias = PK.fold_bn(conv_bias, bn, co, co_pad)
        scale_d, bias_d = self.const(scale), self.const(bias)
        lib = self.lib
        hw = yk.H * yk.W

        def fn_sum(stream):
            L.check(lib.pv_temporal_tap_sum(yk.ptr(), y.ptr(), self.dt, yk.N, Ti, To, hw, co_pad, kt, st, pt, dlt,
                                            scale_d.data_ptr(), bias_d.data_ptr(), act, yk.row_stride,
                                            y.row_stride, stream), "pv_temporal_tap_sum(%s)" % name)
        self.add(name + ".tapsum", fn_sum, "other", 0.0, (yk.N * Ti * hw * kt * co_pad + yk.N * To * hw * co_pad) * 2,
                 reads=(yk,), writes=(y,),
                 spec={"kind": "tap_sum", "x": yk, "y": y, "kt": kt, "st": st, "pt": pt, "dil": dlt, "scale": scale[:co],
                       "bias": bias[:co], "act": act})
        return y

    def _emit_stem_stream(self, x, d, weight, co, lead, name, flops, nbytes):
        """The temporal-streaming stem (csrc/pv_stem_stream.cu) for descriptor ``d``, which the library accepted: the
        temporal sum of the convolution, without BN (unit scale, zero bias) and activation (d.act = none)."""
        self.materialize_input(x, w_pad=d.x_w_pad, w_phys=d.x_w_phys)
        y = self.new_tensor(x.N, d.To, d.Ho, d.Wo, co, Cp=d.Co)
        scale, bias = PK.fold_bn(None, None, co, d.Co)
        scale_d, bias_d = self.const(scale), self.const(bias)
        w_d = self.const(PK.pack_stem_stream(weight, x.Cp, d.Co, lead))
        zero_row = self.const(torch.zeros(4096, dtype=torch.float16))
        lib = self.lib

        def fn(stream):
            d.x_row_stride, d.y_row_stride = x.row_stride, y.row_stride   # y may have been retargeted
            L.check(lib.pv_conv3d_stem_stream_fwd(C.byref(d), x.ptr(), w_d.data_ptr(), scale_d.data_ptr(),
                                                  bias_d.data_ptr(), zero_row.data_ptr(), y.ptr(), stream),
                    "pv_conv3d_stem_stream_fwd(%s)" % name)
        self.stats["stem_stream"] = self.stats.get("stem_stream", 0) + 1
        self.add(name, fn, "tcgen05", flops, nbytes, reads=(x,), writes=(y,),
                 spec={"kind": "conv", "route": "stem_stream", "x": x, "weight": weight, "scale": scale[:co],
                       "bias": bias[:co], "stride": (d.st, d.sh, d.sw), "padding": (d.pt, d.ph, d.pw),
                       "dilation": (d.dt, d.dh, d.dw), "groups": 1, "act": L.ACT_NONE, "residual": None, "addend": None,
                       "y": y, "se_sums": None})
        return y

    def _conv_desc(self, x, out_thw, co_pad, kernel, stride, padding, dilation, groups, act, residual, y_row_stride,
                   ci_pad64):
        d = L.Conv3dDesc()
        d.dtype = self.dt
        d.N, d.Ti, d.Hi, d.Wi, d.Ci = x.N, x.T, x.H, x.W, x.Cp
        d.To, d.Ho, d.Wo = out_thw
        d.Co = co_pad
        d.kt, d.kh, d.kw = kernel
        d.st, d.sh, d.sw = stride
        d.pt, d.ph, d.pw = padding
        d.dt, d.dh, d.dw = dilation
        d.groups = groups
        d.act = act
        d.has_residual = 1 if residual is not None else 0
        d.x_row_stride, d.y_row_stride = x.row_stride, y_row_stride
        d.res_row_stride = residual.row_stride if residual is not None else 0
        d.ci_pad64 = ci_pad64
        return d

    def fused_bottleneck_desc(self, x, cin_pad, cmid, cout, kt, sb, has_shortcut, act):
        d = L.BottleneckDesc()
        d.N, d.T, d.H, d.W = x.N, x.T, x.H, x.W
        d.Cin, d.Cmid, d.Cout = cin_pad, PK.pad8(cmid), PK.pad8(cout)
        d.kt, d.sb, d.has_shortcut, d.act = kt, sb, 1 if has_shortcut else 0, act
        d.x_row_stride, d.y_row_stride = x.row_stride, PK.pad8(cout)
        return d

    def emit_bottleneck_fused(self, x, conv_a, bn_a, conv_b, bn_b, conv_c, bn_c, sc_conv, sc_bn, act, name):
        """ONE launch for conv_a -> conv_b -> conv_c (+ projection / identity shortcut) + activation
        (csrc/pv_fastblock.cu); the caller has checked eligibility with pv_bottleneck_fused_supported."""
        self.materialize_input(x)
        kt, sb = int(conv_a.kernel_size[0]), int(conv_b.stride[1])
        cmid, cout = conv_a.out_channels, conv_c.out_channels
        d = self.fused_bottleneck_desc(x, x.Cp, cmid, cout, kt, sb, sc_conv is not None, act)
        Ho, Wo = (x.H - 1) // sb + 1, (x.W - 1) // sb + 1
        y = self.new_tensor(x.N, x.T, Ho, Wo, cout, Cp=d.Cout)
        wa = self.const(PK.pack_rows_k16(conv_a.weight, x.Cp, d.Cmid))
        wb = self.const(PK.pack_rows_k16(conv_b.weight, d.Cmid, d.Cmid))
        wc = self.const(PK.pack_rows_k16(conv_c.weight, d.Cmid, d.Cout))
        ws = self.const(PK.pack_rows_k16(sc_conv.weight, x.Cp, d.Cout)) if sc_conv is not None else None
        folds = (PK.fold_bn(conv_a.bias, bn_a, cmid, d.Cmid), PK.fold_bn(conv_b.bias, bn_b, cmid, d.Cmid),
                 PK.fold_bn(conv_c.bias, bn_c, cout, d.Cout),
                 PK.fold_bn(sc_conv.bias, sc_bn, cout, d.Cout) if sc_conv is not None else (None, None))
        sa, ba = (self.const(t) for t in folds[0])
        sbb, bbb = (self.const(t) for t in folds[1])
        scc, bcc = (self.const(t) for t in folds[2])
        ss, bs = (self.const(t) for t in folds[3]) if sc_conv is not None else (None, None)
        lib = self.lib

        def fn(stream):
            d.x_row_stride, d.y_row_stride = x.row_stride, y.row_stride
            L.check(lib.pv_bottleneck_fused_fwd(C.byref(d), x.ptr(), wa.data_ptr(), wb.data_ptr(), wc.data_ptr(),
                                                ws.data_ptr() if ws is not None else None, sa.data_ptr(), ba.data_ptr(),
                                                sbb.data_ptr(), bbb.data_ptr(), scc.data_ptr(), bcc.data_ptr(),
                                                ss.data_ptr() if ss is not None else None,
                                                bs.data_ptr() if bs is not None else None, y.ptr(), stream),
                    "pv_bottleneck_fused_fwd(%s)" % name)
        m_in, m_out = x.N * x.T * x.H * x.W, x.N * x.T * Ho * Wo
        cin = conv_a.in_channels
        flops = 2.0 * (m_in * cmid * cin * kt + m_out * cmid * cmid * 9 + m_out * cout * cmid +
                       (m_out * cout * cin if sc_conv is not None else 0))
        nbytes = (m_in * cin + m_out * cout) * 2 + sum(t.numel() for t in (wa, wb, wc)) * 2
        widths = (cmid, cmid, cout, cout)
        self.add(name, fn, "fused_block", flops, nbytes, reads=(x,), writes=(y,),
                 spec={"kind": "fused_block", "x": x, "y": y, "wa": conv_a.weight, "wb": conv_b.weight,
                       "wc": conv_c.weight, "ws": sc_conv.weight if sc_conv is not None else None, "kt": kt, "sb": sb,
                       "act": act, "folds": tuple(None if t is None else t[:c] for f, c in zip(folds, widths) for t in f),
                       "modules": (conv_a, conv_b, conv_c, sc_conv)})
        return y

    def emit_pool(self, x, mode, kernel, stride, padding, name="pool"):
        self.materialize_input(x)
        kt, kh, kw = kernel
        st, sh, sw = stride
        pt, ph, pw = padding
        To, Ho, Wo = (x.T + 2 * pt - kt) // st + 1, (x.H + 2 * ph - kh) // sh + 1, (x.W + 2 * pw - kw) // sw + 1
        if min(To, Ho, Wo) <= 0:
            raise RuntimeError("pool %s: kernel %s larger than input (%d,%d,%d)" % (name, kernel, x.T, x.H, x.W))
        y = self.new_tensor(x.N, To, Ho, Wo, x.C, Cp=x.Cp)
        d = L.Pool3dDesc()
        d.dtype, d.mode = self.dt, mode
        d.N, d.Ti, d.Hi, d.Wi, d.C = x.N, x.T, x.H, x.W, x.Cp
        d.To, d.Ho, d.Wo = To, Ho, Wo
        d.kt, d.kh, d.kw, d.st, d.sh, d.sw, d.pt, d.ph, d.pw = kt, kh, kw, st, sh, sw, pt, ph, pw
        lib = self.lib

        def fn(stream):
            d.x_row_stride, d.y_row_stride = x.row_stride, y.row_stride
            L.check(lib.pv_pool3d_fwd(C.byref(d), x.ptr(), y.ptr(), stream), "pv_pool3d_fwd(%s)" % name)
        self.add(name, fn, reads=(x,), writes=(y,),
                 spec={"kind": "pool", "x": x, "y": y, "mode": mode, "kernel": tuple(kernel), "stride": tuple(stride),
                       "padding": tuple(padding), "cls": 0})
        return y

    def emit_se_scale_act(self, x, w1, b1, w2, b2, act, name="se"):
        """In-place y = act(x * sigmoid(W2 relu(W1 mean(x) + b1) + b2)) (fvcore SqueezeExcitation)."""
        Cr, Cc = w1.shape[0], w1.shape[1]
        assert Cc == x.C
        Cp = x.Cp
        w1p = torch.zeros(Cr, Cp, dtype=torch.float32)
        w1p[:, :Cc] = w1.detach().float().cpu().reshape(Cr, Cc)
        w2p = torch.zeros(Cp, Cr, dtype=torch.float32)
        w2p[:Cc] = w2.detach().float().cpu().reshape(Cc, Cr)
        b2p = torch.zeros(Cp, dtype=torch.float32)
        b2p[:Cc] = b2.detach().float().cpu()
        w1d, b1d, w2d, b2d = self.const(w1p), self.const(b1.detach().float().cpu()), self.const(w2p), self.const(b2p)
        fused = getattr(x, "se_sums", None)       # already produced by the depthwise conv kernel
        sums = fused if fused is not None else self.new_buf(2 * x.N * Cp, L.PV_F32)   # int64 fixed point per (n, c)
        gate = self.new_buf(x.N * Cp, L.PV_F32)
        if fused is None:
            self.zero_bufs.append(sums)
        lib = self.lib
        npos = x.npos

        def fn_sum(stream):
            L.check(lib.pv_zero_f32(sums.tensor.data_ptr(), 2 * x.N * Cp, stream), "pv_zero_f32")
            L.check(lib.pv_channel_sum(x.ptr(), x.dt, x.row_stride, x.N, npos, Cp, sums.tensor.data_ptr(), stream),
                    "pv_channel_sum(%s)" % name)

        def fn_gate(stream):
            L.check(lib.pv_se_gate(sums.tensor.data_ptr(), npos, x.N, Cp, Cr, w1d.data_ptr(), b1d.data_ptr(),
                                   w2d.data_ptr(), b2d.data_ptr(), Cp, gate.tensor.data_ptr(), stream),
                    "pv_se_gate(%s)" % name)

        def fn_apply(stream):
            L.check(lib.pv_scale_act(x.ptr(), x.ptr(), x.dt, x.row_stride, x.row_stride, x.N, npos, Cp,
                                     gate.tensor.data_ptr(), act, stream), "pv_scale_act(%s)" % name)
        if fused is None:
            self.add(name + ".sum", fn_sum, reads=(x,), writes=(sums,), spec={"kind": "channel_sum", "x": x, "sums": sums})
        self.add(name + ".gate", fn_gate, reads=(sums,), writes=(gate,),
                 spec={"kind": "se_gate", "x": x, "sums": sums, "gate": gate, "w1": w1p[:, :Cc],
                       "b1": b1.detach().float().cpu(), "w2": w2p[:Cc], "b2": b2p[:Cc]})
        self.add(name + ".apply", fn_apply, reads=(x, gate), writes=(x,),
                 spec={"kind": "scale_act", "x": x, "y": x, "gate": gate, "act": act})
        return x

    def raw_input(self, static_in):
        """A plan input that is used as it is (fp32 device tensor, no layout / dtype conversion): the [K, 5] bounding
        boxes of the detection heads.  The handle carries the static tensor; ops read its data pointer at run time."""
        return RawIn(static_in)

    def emit_roi_align(self, x, rois, output_size, spatial_scale, sampling_ratio, name="roi_align"):
        """torchvision RoIAlign (aligned=False) on a T == 1 feature map (models/head.py:462-471): [N,1,H,W,C] x
        [K,5] -> [K,1,R_h,R_w,C]."""
        if x.T != 1:
            raise RuntimeError("Temporal dimension should be 1. Consider modifying the pool layer.")   # head.py:464-467
        self.materialize_input(x)
        K = int(rois.tensor.shape[0])
        rh, rw = int(output_size[0]), int(output_size[1])
        y = self.new_tensor(K, 1, rh, rw, x.C, Cp=x.Cp)
        lib = self.lib
        N, H, W, Cp = x.N, x.H, x.W, x.Cp

        def fn(stream):
            L.check(lib.pv_roi_align_fwd(x.ptr(), x.dt, x.row_stride, N, H, W, Cp, rois.tensor.data_ptr(), K, rh, rw,
                                         float(spatial_scale), int(sampling_ratio), y.ptr(), y.row_stride, stream),
                    "pv_roi_align_fwd(%s)" % name)
        self.add(name, fn, reads=(x,), writes=(y,), spec={"kind": "roi_align", "x": x, "rois": rois, "y": y,
                                                          "geom": (rh, rw, float(spatial_scale), int(sampling_ratio))})
        return y

    def emit_act(self, x, act, name="act"):
        lib = self.lib

        def fn(stream):
            L.check(lib.pv_scale_act(x.ptr(), x.ptr(), x.dt, x.row_stride, x.row_stride, x.N, x.npos, x.Cp,
                                     None, act, stream), "pv_scale_act(%s)" % name)
        self.add(name, fn, reads=(x,), writes=(x,), spec={"kind": "scale_act", "x": x, "y": x, "gate": None, "act": act})
        return x

    def emit_head_reduce(self, x, softmax, name="head_reduce"):
        out = self.new_buf(x.N * x.C, L.PV_F32)
        lib = self.lib

        def fn(stream):
            L.check(lib.pv_head_reduce(x.ptr(), x.dt, x.row_stride, x.N, x.npos, x.C, 1 if softmax else 0,
                                       out.tensor.data_ptr(), stream), "pv_head_reduce(%s)" % name)
        self.add(name, fn, reads=(x,), writes=(out,), spec={"kind": "head_reduce", "x": x, "out": out, "softmax": softmax})
        return out, (x.N, x.C)

    def emit_to_ncdhw(self, x, name="to_ncdhw"):
        self.materialize_input(x)
        out = self.new_buf(x.N * x.C * x.npos, L.PV_F32)
        lib = self.lib

        def fn(stream):
            L.check(lib.pv_ndhwc_to_ncdhw(x.ptr(), x.dt, x.row_stride, out.tensor.data_ptr(), x.N, x.C, x.T,
                                          x.H, x.W, stream), "pv_ndhwc_to_ncdhw(%s)" % name)
        self.add(name, fn, reads=(x,), writes=(out,), spec={"kind": "to_f32", "x": x, "out": out, "layout": "ncdhw"})
        return out, x.shape5()

    def emit_input_tokens(self, static_in):
        """static_in: torch tensor [B, N, C] (or [B, C]) f32|f16, contiguous: token-major network input
        (the layout MViT blocks exchange).  One cast/copy launch into the plan's dtype."""
        shp = tuple(static_in.shape)
        B, N, Cc = (shp[0], 1, shp[1]) if len(shp) == 2 else shp
        if Cc % 8 and self.dt == L.PV_F16 and len(shp) == 2:
            # (batch, feature) rows of any width (the projector MLPs of the self-supervised models): rows padded to a
            # multiple of 8 with zero channels, the layout of a (B, C, 1, 1, 1) clip
            return self.materialize_input(self.emit_input_ncdhw(static_in.view(B, Cc, 1, 1, 1), Cc, PK.pad8(Cc)))
        if Cc % 8 and self.dt == L.PV_F16:
            raise RuntimeError("token width %d is not a multiple of 8 (16-byte rows are required in f16 mode)" % Cc)
        x = self.new_tensor(B, 1, 1, N, Cc, Cp=Cc)
        src_dt = L.PV_F32 if static_in.dtype == torch.float32 else L.PV_F16
        total = B * N * Cc
        lib = self.lib

        def fn(stream):
            # a [1, 1, 1, 1, total] "clip" with one channel: the layout conversion degenerates to a cast
            L.check(lib.pv_ncdhw_to_ndhwc(static_in.data_ptr(), src_dt, x.ptr(), x.dt, 1, 1, 1, 1, total, 1, 1, stream),
                    "pv_ncdhw_to_ndhwc(tokens)")
        self.add("tokens_in", fn, "other", 0.0, total * (static_in.element_size() + _ESIZE[self.dt]), reads=(), writes=(x,),
                 spec={"kind": "tokens_in", "src": static_in, "y": x})
        return x

    def emit_to_tokens(self, x, name="to_tokens", squeeze=False):
        """Token TRef [B, N, C] -> f32 output buffer laid out (B, N, C) (or (B, C) with squeeze)."""
        self.materialize_input(x)
        lib = self.lib
        if x.npos == 1 and x.C % 8 and (x.row_stride != x.C or x.Cp != x.C):
            # padded (B, C) rows narrower than a 16-byte vector (the projector outputs of the self-supervised models),
            # which pv_copy_rows does not take: the NDHWC -> NCDHW conversion of (B, C, 1, 1, 1) drops the pad
            # channels on the way out
            out = self.new_buf(x.N * x.C, L.PV_F32)
            src = x

            def fn_r(stream):
                L.check(lib.pv_ndhwc_to_ncdhw(src.ptr(), src.dt, src.row_stride, out.tensor.data_ptr(), src.N, src.C, 1,
                                              1, 1, stream), "pv_ndhwc_to_ncdhw(%s)" % name)
            self.add(name, fn_r, reads=(src,), writes=(out,),
                     spec={"kind": "to_f32", "x": src, "out": out, "layout": "ncdhw"})
            return out, ((x.N, x.C) if squeeze else (x.N, 1, x.C))
        if x.row_stride != x.C or x.Cp != x.C:
            dense = self.new_tensor(x.N, 1, 1, x.npos, x.C, Cp=x.C, dt=x.dt)
            src = x

            def fn_c(stream):
                L.check(lib.pv_copy_rows(src.ptr(), dense.ptr(), src.dt, src.N * src.npos, src.C, src.row_stride,
                                         dense.row_stride, stream), "pv_copy_rows(%s)" % name)
            self.add(name + ".dense", fn_c, reads=(src,), writes=(dense,), spec={"kind": "copy", "x": src, "y": dense})
            x = dense
        total = x.N * x.npos * x.C
        out = self.new_buf(total, L.PV_F32)

        def fn(stream):
            L.check(lib.pv_ndhwc_to_ncdhw(x.ptr(), x.dt, 1, out.tensor.data_ptr(), 1, 1, 1, 1, total, stream),
                    "pv_ndhwc_to_ncdhw(%s)" % name)
        self.add(name, fn, reads=(x,), writes=(out,), spec={"kind": "to_f32", "x": x, "out": out, "layout": "ndhwc"})
        return out, ((x.N, x.C) if squeeze and x.npos == 1 else (x.N, x.npos, x.C))

    def concat_channels(self, parts):
        """Fuse torch.cat(parts, dim=1): retarget every part into one wide buffer (no copy)."""
        p0 = parts[0]
        for p in parts:
            assert (p.N, p.T, p.H, p.W) == (p0.N, p0.T, p0.H, p0.W), "concat shape mismatch"
            assert p.C == p.Cp or p is parts[-1], "only the last concat part may carry channel padding"
        c_total = sum(p.C for p in parts)
        cp_total = PK.pad8(sum(p.Cp for p in parts[:-1]) + parts[-1].Cp)
        buf = self.new_buf(p0.N * p0.npos * cp_total)
        off = 0
        for p in parts:
            p.retarget(buf, off, cp_total)
            off += p.Cp
        return TRef(buf, p0.N, p0.T, p0.H, p0.W, c_total, Cp=cp_total, ch_off=0, row_stride=cp_total)


# =============================================================================================
# Token-major (MViT) emitters.  A token tensor [B, Ntok, C] is a TRef with T=H=1, W=Ntok.
# =============================================================================================
def _tok(plan, B, ntok, C, dt=None):
    return plan.new_tensor(B, 1, 1, ntok, C, Cp=C, dt=dt)


def emit_linear(plan, x, weight, bias, act=L.ACT_NONE, residual=None, name="linear"):
    """nn.Linear on tokens = 1x1x1 convolution (tcgen05 implicit GEMM in f16 mode)."""
    w = weight.reshape(weight.shape[0], weight.shape[1], 1, 1, 1)
    return plan.emit_conv(x, w, bias, None, (1, 1, 1), (0, 0, 0), (1, 1, 1), 1, act, residual, name)


def emit_layernorm(plan, x, ln, name="ln", rows_stride=None, rows=None):
    """LayerNorm over the channel dim of every token (or of `rows` rows spaced rows_stride apart)."""
    C = x.C
    assert tuple(ln.normalized_shape) == (C,), "LayerNorm width mismatch"
    g = plan.const(ln.weight.detach().float().cpu())
    b = plan.const(ln.bias.detach().float().cpu())
    eps = float(ln.eps)
    n_rows = x.N * x.npos if rows is None else rows
    xs = x.row_stride if rows_stride is None else rows_stride
    y = plan.new_tensor(x.N, 1, 1, x.npos if rows is None else 1, C, Cp=C)
    lib = plan.lib
    # rows: the first row of each sample (the cls rows of the MViT head)
    spec = {"kind": "layernorm", "x": x, "y": y, "gamma": ln.weight.detach().float().cpu(),
            "beta": ln.bias.detach().float().cpu(), "eps": eps, "first_row_only": rows is not None}
    if x.dt != plan.dt:          # fp32 trunk of the f16 engine: f32 in, f16 out
        assert x.dt == L.PV_F32 and plan.dt == L.PV_F16

        def fn32(stream):
            L.check(lib.pv_add_layernorm(x.ptr(), x.dt, xs, None, 0, None, 0, y.ptr(), y.row_stride, n_rows, C,
                                         g.data_ptr(), b.data_ptr(), eps, stream), "pv_add_layernorm(%s)" % name)
        plan.add(name, fn32, "other", 0.0, n_rows * C * 6, reads=(x,), writes=(y,), spec=spec)
        return y

    def fn(stream):
        L.check(lib.pv_layernorm(x.ptr(), y.ptr(), x.dt, n_rows, 1, C, xs, y.row_stride, g.data_ptr(), b.data_ptr(),
                                 eps, stream), "pv_layernorm(%s)" % name)
    plan.add(name, fn, "other", 0.0, n_rows * C * 4, reads=(x,), writes=(y,), spec=spec)
    return y


def emit_add_layernorm(plan, a, br, ln, name="add_ln", want_sum=True):
    """fp32 residual trunk of the f16 engine (layers/attention.py:746-757): s = a + br with a f16|f32 and br the f16
    branch output; returns (s as an fp32 token tensor or None, LayerNorm(s) as f16 or None when ln is None)."""
    C = a.C
    assert br.C == C and br.N == a.N and br.npos == a.npos, "residual / branch shape mismatch"
    assert br.dt == L.PV_F16 and plan.dt == L.PV_F16
    assert want_sum or ln is not None
    n_rows = a.N * a.npos
    s = _tok(plan, a.N, a.npos, C, dt=L.PV_F32) if want_sum else None
    y = g = b = None
    eps = 0.0
    if ln is not None:
        assert tuple(ln.normalized_shape) == (C,), "LayerNorm width mismatch"
        g = plan.const(ln.weight.detach().float().cpu())
        b = plan.const(ln.bias.detach().float().cpu())
        eps = float(ln.eps)
        y = _tok(plan, a.N, a.npos, C)
    lib = plan.lib

    def fn(stream):
        L.check(lib.pv_add_layernorm(a.ptr(), a.dt, a.row_stride, br.ptr(), br.row_stride,
                                     s.ptr() if s is not None else None, s.row_stride if s is not None else 0,
                                     y.ptr() if y is not None else None, y.row_stride if y is not None else 0,
                                     n_rows, C, g.data_ptr() if g is not None else None,
                                     b.data_ptr() if b is not None else None, eps, stream), "pv_add_layernorm(%s)" % name)
    plan.add(name, fn, "other", 0.0, n_rows * C * (_ESIZE[a.dt] + 2 + (4 if want_sum else 0) + (2 if ln is not None else 0)),
             reads=(a, br), writes=tuple(t for t in (s, y) if t is not None), spec={"kind": "add_layernorm", "a": a, "br": br, "s": s, "y": y, "eps": eps,
                   "gamma": ln.weight.detach().float().cpu() if ln is not None else None,
                   "beta": ln.bias.detach().float().cpu() if ln is not None else None})
    return s, y


def emit_pos_cls(plan, x, pos_table, has_cls, name="posenc", out_dt=None):
    """x: patch tokens as produced by the patch-embed conv [B, T', H', W', C] -> [B, cls+THW, C] (out_dt = PV_F32
    starts the fp32 residual trunk of the f16 engine)."""
    n_patch = x.npos
    C = x.C
    pos = plan.const(pos_table.float().contiguous())
    y = _tok(plan, x.N, n_patch + (1 if has_cls else 0), C, dt=out_dt)
    lib = plan.lib

    def fn(stream):
        L.check(lib.pv_add_pos_cls_to(x.ptr(), x.dt, y.ptr(), y.dt, x.N, n_patch, C, x.row_stride, pos.data_ptr(),
                                      1 if has_cls else 0, stream), "pv_add_pos_cls_to")
    plan.add(name, fn, "other", 0.0, x.N * n_patch * C * (_ESIZE[x.dt] + _ESIZE[y.dt]), reads=(x,), writes=(y,),
             spec={"kind": "pos_cls", "x": x, "y": y, "pos": pos_table.float(), "has_cls": bool(has_cls)})
    return y


def _pool_geometry(pool):
    kind = type(pool).__name__
    if kind == "Conv3d":
        k, s, p, dl = [tuple(int(v) for v in t) for t in (pool.kernel_size, pool.stride, pool.padding, pool.dilation)]
        return kind, k, s, p, dl, int(pool.in_channels)
    if kind in ("MaxPool3d", "AvgPool3d"):
        if kind == "AvgPool3d" and (pool.ceil_mode or not pool.count_include_pad or pool.divisor_override is not None):
            raise NotImplementedError("AvgPool3d pools take count_include_pad=True, ceil_mode=False and no divisor_override")
        k, s, p = [tuple(int(v) for v in (t if isinstance(t, (tuple, list)) else (t,) * 3))
                   for t in (pool.kernel_size, pool.stride, pool.padding)]
        return kind, k, s, p, (1, 1, 1), 0
    raise NotImplementedError("pool module %s unsupported" % kind)


def bn_affine(bn):
    """Eval-mode BatchNorm as a per-channel affine (scale, shift), fp32 CPU tensors."""
    if bn.running_mean is None or bn.running_var is None:
        raise NotImplementedError("BatchNorm without running statistics is unsupported")
    with torch.no_grad():
        inv = 1.0 / torch.sqrt(bn.running_var.detach().double().cpu() + float(bn.eps))
        w = bn.weight.detach().double().cpu() if bn.weight is not None else torch.ones_like(inv)
        b = bn.bias.detach().double().cpu() if bn.bias is not None else torch.zeros_like(inv)
        s = w * inv
        return s.float(), (b - bn.running_mean.detach().double().cpu() * s).float()


def _prologue_vectors(norm, width):
    """_AttentionPool with norm_before_pool (layers/attention.py:191-195): GELU(norm(x)) before the pool.  BatchNorm3d
    (eval) gives its affine, Identity the unit one; (scale, shift) of ``width`` channels."""
    kind = type(norm).__name__
    if kind == "BatchNorm3d":
        s, b = bn_affine(norm)
        if s.numel() != width:
            raise RuntimeError("attention-pool BatchNorm3d has %d channels, the pool %d" % (s.numel(), width))
        return s, b
    if kind == "Identity":
        return torch.ones(width), torch.zeros(width)
    raise NotImplementedError("pre-pool norm %s unsupported" % kind)


def pools_fusable(pool_a, pool_b, norm_a, norm_b, before_a=False, before_b=False):
    """True when two _AttentionPool branches (pool_k / pool_v) can run as ONE depthwise launch over adjacent channel
    slices: same conv geometry, and either LayerNorms of the same width / eps after the pool (then ONE LayerNorm launch
    for both) or a pre-pool norm + GELU on both (the prologue vectors are concatenated over the two slices)."""
    if type(pool_a).__name__ != "Conv3d" or type(pool_b).__name__ != "Conv3d":
        return False
    if _pool_geometry(pool_a) != _pool_geometry(pool_b):
        return False
    if before_a or before_b:
        return before_a and before_b
    na, nb = type(norm_a).__name__, type(norm_b).__name__
    if na != "LayerNorm" or nb != "LayerNorm":
        return False
    return tuple(norm_a.normalized_shape) == tuple(norm_b.normalized_shape) and float(norm_a.eps) == float(norm_b.eps)


def emit_token_pool(plan, x, thw, pool, norm, heads, has_cls, name="pool", norm_before_pool=False):
    """_AttentionPool (layers/attention.py:162-212) on a token tensor/slice x [B, cls+THW, dim]:
    depthwise Conv3d / MaxPool3d / AvgPool3d over the (T,H,W) grid of the patch tokens (cls row passes through),
    then the per-head LayerNorm over head_dim (cls row included; it is read straight from x by the LayerNorm
    launch).  With ``norm_before_pool`` (BatchNorm3d or Identity norms) the norm and a GELU run instead as the
    prologue of the depthwise conv, on every in-bounds input before the zero padding, and the cls row is copied raw.
    ``pool`` / ``norm`` may be tuples (pool_k, pool_v) / (norm_k, norm_v): x then holds the branches as
    adjacent channel slices and both run in one depthwise (+ one LayerNorm) launch (see pools_fusable).
    Returns (tokens, thw')."""
    import ctypes as C_
    pools = list(pool) if isinstance(pool, (tuple, list)) else [pool]
    norms = list(norm) if isinstance(norm, (tuple, list)) else [norm] * len(pools)
    nset = len(pools)
    T, H, W = thw
    dim_all = x.C
    assert dim_all % nset == 0
    dim = dim_all // nset
    cls = 1 if has_cls else 0
    assert x.npos == cls + T * H * W, "token count does not match thw"
    kind, k, s, p, dl, pool_ch = _pool_geometry(pools[0])
    for q in pools[1:]:
        assert _pool_geometry(q) == (kind, k, s, p, dl, pool_ch)
    if kind == "Conv3d":
        for q in pools:
            if q.groups != q.in_channels or q.in_channels != q.out_channels or q.bias is not None:
                raise NotImplementedError("%s: only depthwise, bias-free pooling convs are supported" % name)
        if dim % pool_ch:
            raise RuntimeError("%s: pool channels do not divide the token width" % name)
    elif norm_before_pool:
        raise NotImplementedError("%s: a pre-pool norm needs a pooling conv" % name)
    To = (T + 2 * p[0] - dl[0] * (k[0] - 1) - 1) // s[0] + 1
    Ho = (H + 2 * p[1] - dl[1] * (k[1] - 1) - 1) // s[1] + 1
    Wo = (W + 2 * p[2] - dl[2] * (k[2] - 1) - 1) // s[2] + 1
    y = _tok(plan, x.N, cls + To * Ho * Wo, dim_all, dt=x.dt)
    lib = plan.lib
    esz = _ESIZE[x.dt]
    if kind == "Conv3d":
        reps = dim // pool_ch
        w_full = torch.cat([q.weight.detach().cpu().repeat(reps, 1, 1, 1, 1) for q in pools], 0)   # same filter for every head
        w_d = plan.const(PK.pack_depthwise(w_full, dim_all, _TORCH_DT[x.dt]))
        ones = plan.const(torch.ones(dim_all, dtype=torch.float32))
        zeros = plan.const(torch.zeros(dim_all, dtype=torch.float32))
        d = L.Conv3dDesc()
        d.dtype = x.dt
        d.N, d.Ti, d.Hi, d.Wi, d.Ci = x.N, T, H, W, dim_all
        d.To, d.Ho, d.Wo, d.Co = To, Ho, Wo, dim_all
        d.kt, d.kh, d.kw = k
        d.st, d.sh, d.sw = s
        d.pt, d.ph, d.pw = p
        d.dt, d.dh, d.dw = dl
        d.groups, d.act, d.has_residual = dim_all, L.ACT_NONE, 0
        d.x_row_stride, d.y_row_stride = x.row_stride, y.row_stride
        d.x_batch_stride, d.y_batch_stride = x.npos * x.row_stride, y.npos * y.row_stride
        pre_vec = None
        if norm_before_pool:
            vec = [_prologue_vectors(n, pool_ch) for n in norms]
            pre_vec = [torch.cat([v_[j].repeat(reps) for v_ in vec]).float().contiguous() for j in (0, 1)]
            pre_s, pre_b = plan.const(pre_vec[0]), plan.const(pre_vec[1])
            d.pre_scale, d.pre_bias, d.pre_act = pre_s.data_ptr(), pre_b.data_ptr(), L.ACT_GELU
            plan.stats["pool_prologue"] = plan.stats.get("pool_prologue", 0) + 1
        # a one-frame token grid (image MViT) pooled by a (1,kh,kw) conv: the plane kernel (csrc/pv_dwplane.cu) when it
        # takes the shape; every other pool keeps pv_dwconv3d_fwd
        plane = k[0] == 1 and T == 1 and bool(lib.pv_dwplane_supported(C_.byref(d)))
        if plane:
            plan.stats["dwplane"] = plan.stats.get("dwplane", 0) + 1

        def fn(stream):
            d.x_row_stride, d.y_row_stride = x.row_stride, y.row_stride
            d.x_batch_stride, d.y_batch_stride = x.npos * x.row_stride, y.npos * y.row_stride
            # the batch strides step over the cls row in front of every sample
            xp, yp = x.ptr() + cls * x.row_stride * esz, y.ptr() + cls * y.row_stride * esz
            if plane:
                L.check(lib.pv_dwplane_fwd(C_.byref(d), xp, w_d.data_ptr(), ones.data_ptr(), zeros.data_ptr(), yp,
                                           stream), "pv_dwplane_fwd(%s)" % name)
            else:
                # depthwise entry point: lane-per-channel-pair stencil for 3x3x3 in f16, generic stencil otherwise
                L.check(lib.pv_dwconv3d_fwd(C_.byref(d), xp, w_d.data_ptr(), ones.data_ptr(), zeros.data_ptr(), yp,
                                            None, stream), "pv_dwconv3d_fwd(%s)" % name)
        plan.add(name + ".dwconv", fn, "depthwise", 2.0 * x.N * To * Ho * Wo * dim_all * k[0] * k[1] * k[2],
                 (x.N * T * H * W + x.N * To * Ho * Wo) * dim_all * esz, reads=(x,), writes=(y,),
                 spec={"kind": "token_conv", "x": x, "y": y, "thw": (T, H, W), "cls": cls, "weight": w_full,
                       "stride": s, "padding": p, "dilation": dl, "prologue": norm_before_pool, "modules": pools,
                       "pre_scale": pre_vec[0] if pre_vec else None, "pre_bias": pre_vec[1] if pre_vec else None})
    else:
        d = L.Pool3dDesc()
        d.dtype, d.mode = x.dt, L.POOL_MAX if kind == "MaxPool3d" else L.POOL_AVG
        d.N, d.Ti, d.Hi, d.Wi, d.C = x.N, T, H, W, dim_all
        d.To, d.Ho, d.Wo = To, Ho, Wo
        d.kt, d.kh, d.kw = k
        d.st, d.sh, d.sw = s
        d.pt, d.ph, d.pw = p

        def fn(stream):
            d.x_row_stride, d.y_row_stride = x.row_stride, y.row_stride
            d.x_batch_stride, d.y_batch_stride = x.npos * x.row_stride, y.npos * y.row_stride
            L.check(lib.pv_pool3d_fwd(C_.byref(d), x.ptr() + cls * x.row_stride * esz,
                                      y.ptr() + cls * y.row_stride * esz, stream), "pv_pool3d_fwd(%s)" % name)
        plan.add(name + (".maxpool" if kind == "MaxPool3d" else ".avgpool"), fn, "other", 0.0,
                 (x.N * T * H * W + x.N * To * Ho * Wo) * dim_all * esz, reads=(x,), writes=(y,),
                 spec={"kind": "pool", "x": x, "y": y, "mode": d.mode, "kernel": k, "stride": s, "padding": p,
                       "cls": cls, "thw": (T, H, W), "modules": pools})
    have_norm = [n is not None and type(n).__name__ != "Identity" and not norm_before_pool for n in norms]
    if any(have_norm) and not all(have_norm):
        raise NotImplementedError("%s: fused pooling branches need a norm on every branch" % name)
    if not all(have_norm):
        if cls:
            def fn_cls(stream):
                L.check(lib.pv_copy_rows(x.ptr(), y.ptr(), x.dt, x.N, dim_all, x.npos * x.row_stride, y.npos * y.row_stride,
                                         stream), "pv_copy_rows(%s)" % name)
            plan.add(name + ".cls", fn_cls, reads=(x,), writes=(y,), spec={"kind": "copy_cls", "x": x, "y": y})
        return y, (To, Ho, Wo)
    for n in norms:
        if type(n).__name__ != "LayerNorm":
            raise NotImplementedError("%s: pool norm %s unsupported" % (name, type(n).__name__))
    hd = int(norms[0].normalized_shape[0])
    eps = float(norms[0].eps)
    for n in norms[1:]:
        assert int(n.normalized_shape[0]) == hd and float(n.eps) == eps
    assert dim % hd == 0
    g = plan.const(torch.cat([n.weight.detach().float().cpu() for n in norms]))
    b = plan.const(torch.cat([n.bias.detach().float().cpu() for n in norms]))

    def fn_ln(stream):
        # in place on the pooled rows; the cls row of every sample (row % npos == 0) is read from x: no copy launch
        L.check(lib.pv_layernorm_sets(y.ptr(), y.ptr(), y.dt, y.N * y.npos, dim_all // hd, hd, y.row_stride, y.row_stride,
                                      g.data_ptr(), b.data_ptr(), dim // hd, x.ptr() if cls else None,
                                      x.npos * x.row_stride, y.npos, eps, stream), "pv_layernorm_sets(%s)" % name)
    plan.add(name + ".norm", fn_ln, "other", 0.0, 2 * y.N * y.npos * dim_all * esz,
             reads=((x,) if cls else ()) + (y,), writes=(y,), spec={"kind": "layernorm_sets", "x": x, "y": y, "cls": cls, "head_dim": hd, "eps": eps,
                   "gamma": torch.cat([n.weight.detach().float().cpu() for n in norms]),
                   "beta": torch.cat([n.bias.detach().float().cpu() for n in norms])})
    return y, (To, Ho, Wo)


def emit_attention(plan, q, k, v, heads, scale, residual_pool, name="attn", normalize=0):
    """normalize = 1: the linear mode of pv_attention_fwd (scores * scale / Nk, no softmax)."""
    import ctypes as C_
    B, Nq, Nk, dim = q.N, q.npos, k.npos, q.C
    assert k.C == dim and v.C == dim and v.npos == Nk and dim % heads == 0
    o = _tok(plan, B, Nq, dim)
    d = L.AttentionDesc()
    d.dtype, d.B, d.H, d.Nq, d.Nk, d.D = plan.dt, B, heads, Nq, Nk, dim // heads
    d.scale, d.add_q_residual = float(scale), 1 if residual_pool else 0
    d.normalize = int(normalize)
    lib = plan.lib

    def fn(stream):
        d.q_row_stride, d.k_row_stride, d.v_row_stride, d.o_row_stride = q.row_stride, k.row_stride, v.row_stride, o.row_stride
        d.q_batch_stride, d.k_batch_stride = Nq * q.row_stride, Nk * k.row_stride
        d.v_batch_stride, d.o_batch_stride = Nk * v.row_stride, Nq * o.row_stride
        L.check(lib.pv_attention_fwd(C_.byref(d), q.ptr(), k.ptr(), v.ptr(), o.ptr(), stream), "pv_attention_fwd(%s)" % name)
    plan.add(name, fn, "attention", 4.0 * B * heads * Nq * Nk * (dim // heads),
             (B * Nq * dim * 2 + 2 * B * Nk * dim) * _ESIZE[plan.dt], reads=(q, k, v), writes=(o,),
             spec={"kind": "attention", "q": q, "k": k, "v": v, "o": o, "heads": heads, "scale": d.scale,
                   "residual": bool(residual_pool), "normalize": d.normalize})
    plan.attention_calls.append({"name": name, "B": B, "H": heads, "Nq": Nq, "Nk": Nk, "D": dim // heads,
                                 "scale": d.scale, "normalize": d.normalize, "add_q_residual": d.add_q_residual})
    return o


def emit_channel_affine(plan, x, scale, shift, name="affine"):
    """y = scale[c] * x + shift[c] on every token row (eval BatchNorm1d over the channels of [B, N, C]), as a 1x1x1
    unit-weight depthwise convolution over a [B, 1, 1, N] grid with the affine as its folded scale / bias."""
    import ctypes as C_
    C = x.C
    y = _tok(plan, x.N, x.npos, C, dt=x.dt)
    w_d = plan.const(PK.pack_depthwise(torch.ones(C, 1, 1, 1, 1), C, _TORCH_DT[x.dt]))
    sc = plan.const(scale.float().contiguous())
    sh = plan.const(shift.float().contiguous())
    d = L.Conv3dDesc()
    d.dtype = x.dt
    d.N, d.Ti, d.Hi, d.Wi, d.Ci = x.N, 1, 1, x.npos, C
    d.To, d.Ho, d.Wo, d.Co = 1, 1, x.npos, C
    d.kt = d.kh = d.kw = d.st = d.sh = d.sw = d.dt = d.dh = d.dw = 1
    d.groups, d.act, d.has_residual = C, L.ACT_NONE, 0
    lib = plan.lib

    def fn(stream):
        d.x_row_stride, d.y_row_stride = x.row_stride, y.row_stride
        d.x_batch_stride, d.y_batch_stride = x.npos * x.row_stride, y.npos * y.row_stride
        L.check(lib.pv_dwconv3d_fwd(C_.byref(d), x.ptr(), w_d.data_ptr(), sc.data_ptr(), sh.data_ptr(), y.ptr(), None,
                                    stream), "pv_dwconv3d_fwd(%s)" % name)
    plan.add(name, fn, "depthwise", 2.0 * x.N * x.npos * C, 2 * x.N * x.npos * C * _ESIZE[x.dt], reads=(x,), writes=(y,),
             spec={"kind": "channel_affine", "x": x, "y": y, "scale": scale.float().cpu(),
                   "shift": shift.float().cpu()})
    return y


def channel_slice(x, off, C):
    """View of C channels starting at `off` (no copy)."""
    t = TRef(x.buf, x.N, x.T, x.H, x.W, C, Cp=C, ch_off=x.ch_off + off, row_stride=x.row_stride)
    return t


# =============================================================================================
# Masked sequence ops (models/masked_multistream.py, layers/fusion.py).  Token tensors [B, T, C] with C % 8 == 0;
# masks are MaskRefs or None (every step valid).
# =============================================================================================
def _mask_ptr(mask):
    return mask.ptr() if mask is not None else None


def _mask_io(mask):
    return mask.io() if mask is not None else ()


def _dense8(x, what):
    if x.C % 8 or x.Cp != x.C:
        raise NotImplementedError("%s: feature width %d is not a multiple of 8" % (what, x.C))


def emit_mask_force_first(plan, mask, name="mask_force_first"):
    """mask[:, 0] = True (models/masked_multistream.py:137-141, :309-313) on a copy owned by the plan."""
    out = MaskRef(mask.B, mask.T, buf=plan.new_buf(mask.B * mask.T, L.PV_U8))
    lib = plan.lib

    def fn(stream):
        L.check(lib.pv_mask_force_first(mask.ptr(), out.ptr(), mask.B, mask.T, stream), "pv_mask_force_first(%s)" % name)
    plan.add(name, fn, "other", 0.0, 2 * mask.B * mask.T, reads=mask.io(), writes=out.io(),
             spec={"kind": "mask_force_first", "mask": mask, "out": out})
    return out


def emit_masked_pool(plan, x, mask, mode, name="masked_pool"):
    """MaskedTemporalPooling (:35-93): [B, T, C] -> [B, C] (a token tensor of one position)."""
    _dense8(x, name)
    y = _tok(plan, x.N, 1, x.C)
    lib = plan.lib
    B, T, Cc = x.N, x.npos, x.C

    def fn(stream):
        L.check(lib.pv_masked_pool(x.ptr(), x.dt, x.row_stride, B, T, Cc, _mask_ptr(mask), mode, y.ptr(), y.row_stride,
                                   stream), "pv_masked_pool(%s)" % name)
    plan.add(name, fn, "other", 0.0, (B * T + B) * Cc * _ESIZE[x.dt], reads=(x,) + _mask_io(mask), writes=(y,),
             spec={"kind": "masked_pool", "x": x, "mask": mask, "mode": mode, "y": y})
    return y


def emit_masked_default(plan, x, mask, default, name="learned_default"):
    """LearnMaskedDefault (:170-190) on [B, C]."""
    _dense8(x, name)
    if x.npos != 1:
        raise NotImplementedError("%s: LearnMaskedDefault on a (batch, seq_len, feature) tensor is unsupported" % name)
    if mask is None:
        raise RuntimeError("%s: LearnMaskedDefault needs a mask" % name)
    d = plan.const(default.detach().float().cpu().reshape(-1))
    if d.numel() != x.C:
        raise RuntimeError("%s: default of %d values for %d features" % (name, d.numel(), x.C))
    y = _tok(plan, x.N, 1, x.C)
    lib = plan.lib

    def fn(stream):
        L.check(lib.pv_masked_default(x.ptr(), x.dt, x.row_stride, x.N, x.C, mask.ptr(), mask.T, d.data_ptr(), y.ptr(),
                                      y.row_stride, stream), "pv_masked_default(%s)" % name)
    plan.add(name, fn, "other", 0.0, 2 * x.N * x.C * _ESIZE[x.dt], reads=(x,) + mask.io(), writes=(y,),
             spec={"kind": "masked_default", "x": x, "mask": mask, "y": y,
                   "default": default.detach().float().cpu().reshape(-1)})
    return y


def emit_reduce_fusion(plan, parts, op, name="reduce_fusion"):
    """ReduceFusion (layers/fusion.py:104-141): elementwise max / sum / prod over P same-shaped token tensors."""
    p0 = parts[0]
    if len(parts) > 8:
        raise NotImplementedError("%s: %d inputs (at most 8)" % (name, len(parts)))
    for p in parts:
        _dense8(p, name)
        if (p.N, p.npos, p.C) != (p0.N, p0.npos, p0.C):
            raise RuntimeError("%s: inputs of different shapes" % name)
    y = _tok(plan, p0.N, p0.npos, p0.C)
    lib = plan.lib
    P = len(parts)
    ptrs, strides = (C.c_void_p * P)(), (C.c_longlong * P)()

    def fn(stream):
        for i, p in enumerate(parts):
            ptrs[i], strides[i] = p.ptr(), p.row_stride
        L.check(lib.pv_reduce_fusion(ptrs, strides, P, p0.dt, p0.N * p0.npos, p0.C, op, y.ptr(), y.row_stride, stream),
                "pv_reduce_fusion(%s)" % name)
    plan.add(name, fn, "other", 0.0, (P + 1) * p0.N * p0.npos * p0.C * _ESIZE[p0.dt], reads=tuple(parts), writes=(y,),
             spec={"kind": "reduce_fusion", "parts": list(parts), "op": op, "y": y})
    return y


def emit_copy_tokens(plan, x, y, row0, name="copy_tokens"):
    """y[b, row0 + i, :] = x[b, i, :] (the row-slice writes of TemporalConcatFusion)."""
    lib = plan.lib

    def fn(stream):
        esz = _ESIZE[x.dt]
        if x.row_stride == x.C and y.row_stride == y.C:
            # dense rows: every sample's rows are one contiguous span, one launch for all samples
            L.check(lib.pv_copy_rows(x.ptr(), y.ptr() + row0 * y.row_stride * esz, x.dt, x.N, x.npos * x.C,
                                     x.npos * x.C, y.npos * y.C, stream), "pv_copy_rows(%s)" % name)
            return
        for b in range(x.N):
            L.check(lib.pv_copy_rows(x.ptr() + b * x.npos * x.row_stride * esz,
                                     y.ptr() + (b * y.npos + row0) * y.row_stride * esz, x.dt, x.npos, x.C,
                                     x.row_stride, y.row_stride, stream), "pv_copy_rows(%s)" % name)
    plan.add(name, fn, "other", 0.0, 2 * x.N * x.npos * x.C * _ESIZE[x.dt], reads=(x,), writes=(y,),
             spec={"kind": "copy_tokens", "x": x, "y": y, "row0": int(row0)})


def emit_attention_masked(plan, q, k, v, heads, scale, mask, name="attn", weights=False):
    """Key-masked softmax attention (pv_attention_masked_fwd) on token tensors; with ``weights`` also the head-averaged
    fp32 softmax [B, Nq, Nk] (pv_attention_weights).  mask None: every key valid.  Returns (o, weights Buf or None)."""
    import ctypes as C_
    B, Nq, Nk, dim = q.N, q.npos, k.npos, q.C
    assert k.C == dim and v.C == dim and v.npos == Nk and dim % heads == 0
    if mask is None:
        mask = MaskRef(B, Nk, tensor=plan.const(torch.ones(B, Nk, dtype=torch.uint8)))
    o = _tok(plan, B, Nq, dim)
    d = L.AttentionDesc()
    d.dtype, d.B, d.H, d.Nq, d.Nk, d.D = plan.dt, B, heads, Nq, Nk, dim // heads
    d.scale, d.add_q_residual, d.normalize = float(scale), 0, 0
    lse = plan.new_buf(B * heads * Nq, L.PV_F32) if weights else None
    w = plan.new_buf(B * Nq * Nk, L.PV_F32) if weights else None
    lib = plan.lib

    def fn(stream):
        d.q_row_stride, d.k_row_stride, d.v_row_stride, d.o_row_stride = q.row_stride, k.row_stride, v.row_stride, o.row_stride
        d.q_batch_stride, d.k_batch_stride = Nq * q.row_stride, Nk * k.row_stride
        d.v_batch_stride, d.o_batch_stride = Nk * v.row_stride, Nq * o.row_stride
        L.check(lib.pv_attention_masked_fwd(C_.byref(d), q.ptr(), k.ptr(), v.ptr(), o.ptr(), mask.ptr(),
                                            lse.tensor.data_ptr() if lse is not None else None, stream),
                "pv_attention_masked_fwd(%s)" % name)
    plan.add(name, fn, "attention", 4.0 * B * heads * Nq * Nk * (dim // heads),
             (B * Nq * dim * 2 + 2 * B * Nk * dim) * _ESIZE[plan.dt], reads=(q, k, v) + mask.io(),
             writes=(o,) + ((lse,) if lse is not None else ()),
             spec={"kind": "attention_masked", "q": q, "k": k, "v": v, "o": o, "heads": heads, "scale": d.scale,
                   "mask": mask, "lse": lse})
    plan.attention_calls.append({"name": name, "B": B, "H": heads, "Nq": Nq, "Nk": Nk, "D": dim // heads,
                                 "scale": d.scale, "normalize": 0, "add_q_residual": 0, "masked": True})
    if weights:
        def fn_w(stream):
            L.check(lib.pv_attention_weights(C_.byref(d), q.ptr(), k.ptr(), mask.ptr(), lse.tensor.data_ptr(),
                                             w.tensor.data_ptr(), stream), "pv_attention_weights(%s)" % name)
        plan.add(name + ".weights", fn_w, "other", 2.0 * B * heads * Nq * Nk * (dim // heads), B * Nq * Nk * 4,
                 reads=(q, k, lse) + mask.io(), writes=(w,),
                 spec={"kind": "attention_weights", "q": q, "k": k, "mask": mask, "lse": lse, "w": w, "heads": heads,
                       "scale": d.scale})
    return o, w
