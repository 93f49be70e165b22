"""Every launch of every model the suite compiles against float64, in f16 and in f32 parity mode.

test_gpu_workload_audit.py audits the seven bench.py workloads in f16.  The other models the engine runs are checked
end to end against the reference's goldens, at bounds loose enough that one wrong tile in one layer disappears after
global average pooling.  This file runs the same per-launch audit (testing.audit_plan) on the whole case catalogue:
every case of MODEL_CASES, HUB_TAIL_CASES, GROUPED_MODEL_CASES, DETECTION_CASES, AUDIO_CASES, EFFICIENT_CASES,
MVIT_VARIANT_CASES, NONLOCAL_CASES and MASKED_CASES plus the I3D-NLN model, in f16 (less the architecture / shape
pairs of the seven workloads and the c1-c4 and *_f16w repeats of other cases) and in f32 parity mode (all of them).
Each case compiles its plan, stages its own inputs, audits clip 0 (batch 1) or clips 0, B // 2 and B - 1 on one
stream, then captures and replays the graph: every plan buffer must equal the single-stream run bit for bit, also
after a replay on other inputs (the clips mirrored along W).  In f32 every comparison uses the fp32 rounding term and
the operands the fp32 kernels read (fp32 weights), and attention the fp32 bound of testing.ACC_EPS_ATTN_F32.

CPU tests: every launch of every case in both precisions has a record the audit checks and the declared I/O covers
it; each new reference and fp32 bound accepts an fp32 emulation of its kernel in the kernel's order of operations and
rejects a named wrong kernel (f16 probabilities in fp32 attention, the linear mode divided by Nq, f16 storage of an
fp32 depthwise or affine result, a GELU prologue applied to the padding, a RoIAlign geometry contracted into FMAs, a
masked average divided by T, swapped LSTM input / forget gates, head weights not averaged).

Measured on an NVIDIA H100 80GB HBM3 (700 W power limit), in three pytest processes of 412 s, 226 s and 229 s (867 s
in all; the longest cases avsf_r50_b8_f16grid 44 s in either precision, mvit_base_32x3 42 s / 41 s):
  f16, 84 cases: 4464 of 4631 launches audited (the other 167 are SE-sum clears).  Largest err / tol per family:
    conv igemm / gather / stem 0.997, grouped 0.994, direct 0.990, depthwise 0.997, fused block 0.752, stem stream
    0.878, temporal tap sum 0.993, average pool 0.991, scale_act 0.999, se_gate 0.005, head 0.014, LayerNorm 0.984 /
    0.987 (sets), add_layernorm 0.985, MViT pooling conv 0.996, channel affine 0.997, attention 0.460, masked
    attention 0.262, attention weights 0.037, RoIAlign 0.998, masked average / sum 0.990, reduce fusion 0.979, LSTM
    0.872.
  f32, 91 cases: 5299 of 5496 launches audited (197 SE-sum clears).  Largest err / tol per family: direct 0.344,
    depthwise 0.365, average pool 0.077, scale_act 0.709, se_gate 0.005, head 0.051, LayerNorm 0.040 / 0.043 (sets),
    MViT pooling conv 0.274, channel affine 0.058, attention 0.039, masked attention 0.019, attention weights 0.038,
    RoIAlign 0.295, masked average / sum 0.030, reduce fusion 0.015, LSTM 0.092.
  Both: layout conversions, copies, token input, mask copies, masked max pooling, learned defaults, max pooling,
  add_pos_cls and the fp32 trunk sums bit-exact; every graph replay equal to the single-stream run in every buffer.
  Self-check (test_f32_audit_names_a_tile_the_parity_tolerance_misses): one 64-row tile of
  blocks.1.res_blocks.0.branch1 moved by 2^-12 relative fails the audit at err / tol 178, while the corrupted logits
  stay within test_model_f32_parity_mode's tolerance (max |d| 2.2e-5).

The audit found no kernel defect.  It found four places where the reference's bound, not the kernel, was incomplete,
each now charged beside its reference in testing.py:
  - avsf_r50 (f16): the tensor-core epilogue adds the audio addend to the f16-rounded result, a second rounding
    (as test_gpu_audio.py's addend rows already allow).
  - i3d_nln (f16): the last res4 Non-local block sees logits up to 2.3e5 (random BatchNorm statistics), where the
    fp32 scores themselves are uncertain by tens; attn_score_extra64 carries the score and __expf error to o.
  - bn_small (f16): a sharp softmax whose winning key has v = 0 leaves o made of probabilities below 2^-14, which f16
    rounds to an absolute step (attn_p16_floor64).
  - x3d_m / x3d_l (f32): pv_channel_sum adds up to a few hundred stored outputs per thread in fp32 before its
    fixed-point atomic (channel_sum_adds); in f16 the storage rounding term had covered it.

test_gpu_batch_audit.py runs the same audit at other batch sizes on every clip, with the SSL / MoCo trunks, and checks
each clip's bits under reordering the batch and against the batch-1 plan.

Not verified: batch sizes other than each case's own and the batch audit's sweep; SM counts other than the test
machine's (the routes read the device's); the transform, bank, contrastive and JPEG kernels (not plan ops); instances
no catalogue case reaches (the kernel matrices cover those per instance); the run time in a single pytest process.
"""
import math
import os
import sys
import time

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from pytorchvideo_b200 import _lib as L  # noqa: E402
from pytorchvideo_b200 import testing as TS  # noqa: E402
from pytorchvideo_b200.engine.plan import Buf, TRef  # noqa: E402

CATALOGUE = TS.audit_catalogue(bench.WORKLOADS)
CASES = TS.audit_cases(bench.WORKLOADS)
IDS = ["%s-%s-%s" % c for c in CASES]
build = TS.build_audit_case


def _flat(x):
    return list(x) if isinstance(x, (list, tuple)) else [x]


# =====================================================================================================================
# GPU: the audit and the graph replay, per case and precision
# =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("prec,family,case", CASES, ids=IDS)
def test_model_audit_and_graph_replay(prec, family, case):
    from pytorchvideo_b200.engine import compile_model
    t0 = time.time()
    m, x, extra, fixed = build(family, case)
    ins = [t.cuda() for t in _flat(x)]
    # the replay's other inputs: every clip / token tensor mirrored along its last axis (masks and boxes kept)
    alt = [t if i in fixed else t.flip(-1).contiguous() for i, t in enumerate(ins)]
    cm = compile_model(m, ins if isinstance(x, (list, tuple)) else ins[0], dtype=prec, use_graph=False, extra=extra)
    plan = cm.plan
    for s, t in zip(cm.static_in, ins):
        s.copy_(t)
    torch.cuda.synchronize()
    B = ins[0].shape[0]
    with torch.no_grad():
        failures, stats = TS.audit_plan(plan, TS.audit_clips(B))
    n_checked = sum(v[0] for v in stats.values())
    insts = set().union(*(v[2] for v in stats.values())) if stats else set()
    assert not failures, "\n".join("op %d %s: %s" % f for f in failures[:20])
    assert n_checked + sum(1 for s in plan.op_spec if s is None) == len(plan.ops)
    lanes, nbufs = TS.check_graph_replay(cm, ins, alt)
    print("RESULT %s %s: %d launches, %d audited, %d instances, replay (%d lanes, %d buffers) equal, %.1f s; "
          "largest err/tol per family: %s" % (
              prec, case, len(plan.ops), n_checked, len(insts), lanes, nbufs, time.time() - t0,
              ", ".join("%s %d x %.4f" % (k, v[0], v[1]) for k, v in sorted(stats.items()))))
    del cm, plan
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_f32_audit_names_a_tile_the_parity_tolerance_misses():
    """f32 x3d_xs: one 64-row tile of one convolution output moved by 2^-12 relative after its launch.  The logits of
    the corrupted run still pass test_model_f32_parity_mode's tolerance against the golden, while the audit fails
    that op and no other."""
    import pytorchvideo_b200.models.hub as PH
    from pytorchvideo_b200.engine import compile_model
    g = torch.load(os.path.join(ROOT, "tests", "golden", "model_x3d_xs.pt"), weights_only=False)
    m, x, _ = TS.build_case("x3d_xs", PH, weight_seed=g["weight_seed"], input_seed=g["input_seed"])
    cm = compile_model(m, x.cuda(), dtype="f32", use_graph=False)
    plan = cm.plan
    target = next(i for i, s in enumerate(plan.op_spec) if s is not None and s["kind"] == "conv"
                  and s["route"] == "direct" and s["y"].N * s["y"].npos >= 4 * 64 and i > 2)

    def corrupt(i, spec):
        if i == target:
            y = spec["y"]
            rows = TS.full_rows(y).reshape(-1, y.row_stride)
            rows[64:128, y.ch_off:y.ch_off + y.C] *= 1 + 2.0 ** -12
    cm.static_in[0].copy_(x.cuda())
    with torch.no_grad():
        failures, _ = TS.audit_plan(plan, TS.audit_clips(x.shape[0]), corrupt=corrupt)
    names = [f[1] for f in failures]
    assert names == [plan.ops[target][0]], failures
    out = cm.output_view().float().cpu()                 # the logits of the corrupted single-stream run
    ref = g["output"]
    scale = max(1.0, float(ref.abs().max()))
    err = (out - ref).abs()
    assert bool((err <= 1e-3 * ref.abs() + 1e-4 * scale).all()), float(err.max())
    print("RESULT f32 self-check: %s rejected (%s); corrupted logits within the parity tolerance (max |d| %.3g)" % (
        names[0], failures[0][2][:100], float(err.max())))


# =====================================================================================================================
# CPU: records and declared I/O over the whole catalogue
# =====================================================================================================================
# every case at its own batch, and every (case, batch) of test_gpu_batch_audit.py's sweep
_RECORD_CASES = [c + (None,) for c in CASES] + [r[:4] for r in TS.batch_sweep(bench.WORKLOADS)]
_RECORD_IDS = IDS + ["%s-%s-%s-b%d" % r[:4] for r in TS.batch_sweep(bench.WORKLOADS)]


@pytest.mark.parametrize("prec,family,case,batch", _RECORD_CASES, ids=_RECORD_IDS)
def test_every_launch_has_a_checked_record(prec, family, case, batch):
    from pytorchvideo_b200.engine.lower import lower_only
    if batch is None:
        m, x, extra, _ = build(family, case)
    else:
        bc = TS.BatchCase(family, case, batch)
        m, x, extra = bc.model, bc.example(bc.batch(batch)), bc.extra
    plan, _ = lower_only(m, x, dtype=prec, extra=extra)
    assert len(plan.op_spec) == len(plan.ops)
    missing = [n for (n, _), s in zip(plan.ops, plan.op_spec)
               if not TS.supported(s) and not n.endswith(TS.NO_VALUE_SUFFIXES)]
    assert not missing, missing
    assert all(s is not None or n.endswith(TS.NO_VALUE_SUFFIXES) for (n, _), s in zip(plan.ops, plan.op_spec))
    for (n, _), s in zip(plan.ops, plan.op_spec):
        if s is not None:
            for t in TS.record_io(s)[0] + TS.record_io(s)[1]:
                assert isinstance(t, (TRef, Buf)), (n, t)
    assert not TS.io_problems(plan)


# =====================================================================================================================
# CPU: the new references and fp32 bounds accept their kernel and reject named wrong kernels
# =====================================================================================================================
def _tok(B, N, C, dt, values):
    """A token TRef [B, N, C] over its own buffer holding ``values``."""
    b = Buf(B * N * C, dt)
    b.tensor = values.to({L.PV_F16: torch.float16, L.PV_F32: torch.float32}[dt]).reshape(-1).clone()
    return TRef(b, B, 1, 1, N, C, Cp=C)


def _fma(a, b, c):
    """fp32 fused multiply-add: the exact product (48 bits) plus c, rounded once to fp32."""
    return (a.double() * b.double() + c.double()).float()


def _attention_f32(q, k, v, scale, p_round=None):
    """The fp32 CUDA-core attention kernel's order of operations (pv_attention.cu) on [B, H, N, D] fp32 operands:
    fmaf dot products of q * scale with k, online softmax over key tiles of 32, fmaf p.v sums, acc * (1 / l).
    p_round: a rounding applied to p before P.V only (a wrong kernel)."""
    B, H, Nq, D = q.shape
    Nk = k.shape[2]
    qs = q * scale
    m = torch.full((B, H, Nq, 1), -math.inf)
    l = torch.zeros(B, H, Nq, 1)
    acc = torch.zeros(B, H, Nq, D)
    for k0 in range(0, Nk, 32):
        kt, vt = k[:, :, k0:k0 + 32], v[:, :, k0:k0 + 32]
        s = torch.zeros(B, H, Nq, kt.shape[2])
        for c in range(D):
            s = _fma(qs[..., c:c + 1], kt[..., c].unsqueeze(2), s)
        m_new = torch.maximum(m, s.max(-1, keepdim=True).values)
        p = torch.exp(s - m_new)
        corr = torch.where(m == -math.inf, torch.zeros_like(m), torch.exp(m - m_new))
        l = l * corr + p.sum(-1, keepdim=True)
        m = m_new
        acc = acc * corr
        pv = p if p_round is None else p_round(p)
        for j in range(kt.shape[2]):
            acc = _fma(pv[..., j:j + 1], vt[:, :, j].unsqueeze(2), acc)
    return acc * (1.0 / l)


def _attn_spec(q, k, v, heads, scale, dt, o, normalize=0):
    """An attention record over token TRefs: q [B, Nq, C], k / v [B, Nk, C], output values o [B, Nq, C]."""
    B, Nq, C = q.shape
    Nk = k.shape[1]
    return {"kind": "attention", "q": _tok(B, Nq, C, dt, q), "k": _tok(B, Nk, C, dt, k), "v": _tok(B, Nk, C, dt, v),
            "o": _tok(B, Nq, C, dt, o), "heads": heads, "scale": scale, "residual": False, "normalize": normalize}


def _audit_one(spec, launched, clips):
    return TS.compare(spec, TS.gather_inputs(spec, clips), clips, launched)


def _rows(t):          # [B, H, N, D] -> [B, N, H * D]
    return t.permute(0, 2, 1, 3).reshape(t.shape[0], t.shape[2], -1)


def _heads(t, H):      # [B, N, H * D] -> [B, H, N, D]
    return t.view(t.shape[0], t.shape[1], H, -1).permute(0, 2, 1, 3)


@pytest.mark.parametrize("D,Nq,Nk,mag", [(32, 40, 33, 3.0), (64, 33, 100, 2.0), (128, 17, 70, 1.0)])
def test_f32_attention_bound_accepts_the_kernel_and_rejects_f16_probabilities(D, Nq, Nk, mag):
    g = torch.Generator().manual_seed(D + Nk)
    B, H = 2, 2
    q, k, v = (torch.randn(B, H, n, D, generator=g) for n in (Nq, Nk, Nk))
    q = q * mag
    scale = D ** -0.5
    launched = {"attention_kernel<float,%d>" % D: 1}
    good = _attention_f32(q, k, v, scale)
    r = _audit_one(_attn_spec(_rows(q), _rows(k), _rows(v), H, scale, L.PV_F32, _rows(good)), launched, [0, 1])
    assert r[0][1] <= 1.0
    bad = _attention_f32(q, k, v, scale, p_round=lambda p: p.half().float())
    with pytest.raises(AssertionError):
        _audit_one(_attn_spec(_rows(q), _rows(k), _rows(v), H, scale, L.PV_F32, _rows(bad)), launched, [0, 1])
    # the f16 bound the kernel matrix used for these rows before does not see the f16 probabilities
    ref, absref = TS.attn_ref64(q, k, v, scale, False)
    TS.assert_close_to_f64(bad, ref, absref, 0, acc_eps=TS.ACC_EPS_ATTN)


def test_f32_linear_attention_bound_accepts_the_kernel_and_rejects_a_wrong_count():
    """normalize = 1 (non-local dot_product): o = (scale q k^T / Nk) v in fp32.  Dividing by Nq instead of Nk fails."""
    g = torch.Generator().manual_seed(5)
    B, H, Nq, Nk, D = 1, 1, 48, 40, 64
    q, k, v = (torch.randn(B, H, n, D, generator=g) for n in (Nq, Nk, Nk))

    def kernel(count):
        s = torch.zeros(B, H, Nq, Nk)
        for c in range(D):
            s = _fma(q[..., c:c + 1], k[..., c].unsqueeze(2), s)
        p = s * (1.0 / count)
        acc = torch.zeros(B, H, Nq, D)
        for j in range(Nk):
            acc = _fma(p[..., j:j + 1], v[:, :, j].unsqueeze(2), acc)
        return acc
    launched = {"attention_kernel<float,64>": 1}
    spec = _attn_spec(_rows(q), _rows(k), _rows(v), H, 1.0, L.PV_F32, _rows(kernel(Nk)), normalize=1)
    assert _audit_one(spec, launched, [0])[0][1] <= 1.0
    with pytest.raises(AssertionError):
        _audit_one(_attn_spec(_rows(q), _rows(k), _rows(v), H, 1.0, L.PV_F32, _rows(kernel(Nq)), normalize=1),
                   launched, [0])


def _dw_spec(x, w, y, stride, padding, dt):
    """A depthwise conv record over NDHWC TRefs: x [N, C, T, H, W], y the output values (same layout)."""
    N, C, T, H, W = x.shape
    xb, yb = Buf(x.numel(), dt), Buf(y.numel(), dt)
    tdt = torch.float32 if dt == L.PV_F32 else torch.float16
    xb.tensor = x.permute(0, 2, 3, 4, 1).to(tdt).reshape(-1).clone()
    yb.tensor = y.permute(0, 2, 3, 4, 1).to(tdt).reshape(-1).clone()
    xt = TRef(xb, N, T, H, W, C, Cp=C)
    yt = TRef(yb, N, *y.shape[2:], C, Cp=C)
    return {"kind": "conv", "route": "depthwise", "x": xt, "weight": w, "scale": torch.ones(C), "bias": torch.zeros(C),
            "stride": stride, "padding": padding, "dilation": (1, 1, 1), "groups": C, "act": L.ACT_NONE,
            "residual": None, "addend": None, "y": yt, "se_sums": None}


def _dw_kernel_f32(x, w, stride, padding):
    """fp32 stencil in tap order: one fmaf per tap."""
    N, C = x.shape[:2]
    kt, kh, kw = w.shape[2:]
    xp = F.pad(x, (padding[2], padding[2], padding[1], padding[1], padding[0], padding[0]))
    To, Ho, Wo = [(xp.shape[2 + i] - w.shape[2 + i]) // stride[i] + 1 for i in range(3)]
    acc = torch.zeros(N, C, To, Ho, Wo)
    for a in range(kt):
        for b in range(kh):
            for c in range(kw):
                tap = xp[:, :, a:a + stride[0] * (To - 1) + 1:stride[0], b:b + stride[1] * (Ho - 1) + 1:stride[1],
                         c:c + stride[2] * (Wo - 1) + 1:stride[2]]
                acc = _fma(tap, w[:, 0, a, b, c].view(1, C, 1, 1, 1), acc)
    return acc


def test_f32_depthwise_bound_rejects_f16_storage():
    g = torch.Generator().manual_seed(11)
    C = 24
    x = torch.randn(2, C, 4, 9, 9, generator=g)
    w = torch.randn(C, 1, 3, 3, 3, generator=g) * 0.3
    s, p = (1, 2, 2), (1, 1, 1)
    y = _dw_kernel_f32(x, w, s, p)
    launched = {"dwconv3d_w4_kernel<float,3,2>": 1}
    assert _audit_one(_dw_spec(x, w, y, s, p, L.PV_F32), launched, [0, 1])[0][1] <= 1.0
    with pytest.raises(AssertionError):
        _audit_one(_dw_spec(x, w, y.half().float(), s, p, L.PV_F32), launched, [0, 1])
    # under the f16 rounding term the f16-stored result would pass
    ref, absref = TS.conv_ref64(x.double(), w.double(), torch.ones(C), torch.zeros(C), s, p, (1, 1, 1), C, None, None)
    TS.assert_close_to_f64(y.half().float(), ref, absref, 27)


def _prologue_case(dt):
    g = torch.Generator().manual_seed(3)
    N, C, T, H = 2, 16, 4, 8
    x = torch.randn(N, 1 + T * H * H, C, generator=g)
    w = torch.randn(C, 1, 3, 3, 3, generator=g) * 0.3
    pre_s, pre_b = torch.rand(C, generator=g) + 0.5, torch.rand(C, generator=g) * 4.0 - 1.0
    return N, C, T, H, x, w, pre_s, pre_b


def _prologue_kernel(x, w, pre_s, pre_b, T, H, pad_value_gelu=False):
    """fp32 prologue conv: u = GELU(fmaf(x, s, b)) on in-bounds taps, zero padding, the fp32 stencil.
    pad_value_gelu: a wrong kernel that applies the prologue to the padding as well."""
    N, _, C = x.shape
    grid = x[:, 1:].reshape(N, T, H, H, C).permute(0, 4, 1, 2, 3)
    pre = _fma(grid, pre_s.view(1, C, 1, 1, 1), pre_b.view(1, C, 1, 1, 1))
    u = (0.5 * pre.double() * (1 + torch.erf(pre.double() / math.sqrt(2.0)))).float()
    if not pad_value_gelu:
        return _dw_kernel_f32(u, w, (1, 2, 2), (1, 1, 1))
    gb = (0.5 * pre_b.double() * (1 + torch.erf(pre_b.double() / math.sqrt(2.0)))).float().view(1, C, 1, 1, 1)
    padded = gb.expand(N, C, T + 2, H + 2, H + 2).clone()
    padded[:, :, 1:-1, 1:-1, 1:-1] = u
    return _dw_kernel_f32(padded, w, (1, 2, 2), (0, 0, 0))


@pytest.mark.parametrize("wrong", [False, True])
def test_prologue_reference_accepts_the_kernel_and_rejects_a_gelu_padding(wrong):
    N, C, T, H, x, w, pre_s, pre_b = _prologue_case(L.PV_F32)
    y = _prologue_kernel(x, w, pre_s, pre_b, T, H, pad_value_gelu=wrong)
    To, Ho = y.shape[2], y.shape[3]
    yrows = torch.cat([torch.zeros(N, 1, C), y.permute(0, 2, 3, 4, 1).reshape(N, -1, C)], 1)
    spec = {"kind": "token_conv", "x": _tok(N, 1 + T * H * H, C, L.PV_F32, x), "y": _tok(N, 1 + To * Ho * Ho, C,
                                                                                         L.PV_F32, yrows),
            "thw": (T, H, H), "cls": 1, "weight": w, "stride": (1, 2, 2), "padding": (1, 1, 1),
            "dilation": (1, 1, 1), "prologue": True, "pre_scale": pre_s, "pre_bias": pre_b}
    launched = {"dwconv3d_w4_kernel<float,3,2>": 1}
    if wrong:
        with pytest.raises(AssertionError):
            _audit_one(spec, launched, [0, 1])
    else:
        assert _audit_one(spec, launched, [0, 1])[0][1] <= 1.0


@pytest.mark.parametrize("dt", [L.PV_F16, L.PV_F32])
def test_copies_and_conversions_are_bit_exact(dt):
    """to_f32, copy, tokens_in: equal bit for bit; one element off by an ulp fails."""
    g = torch.Generator().manual_seed(1)
    B, N, C = 3, 5, 16
    vals = torch.randn(B, N, C, generator=g)
    tdt = torch.float16 if dt == L.PV_F16 else torch.float32
    x = _tok(B, N, C, dt, vals)
    out = Buf(B * N * C, L.PV_F32)
    out.tensor = vals.to(tdt).float().reshape(-1).clone()
    y = _tok(B, N, C, dt, vals)
    specs = [{"kind": "to_f32", "x": x, "out": out, "layout": "ndhwc"}, {"kind": "copy", "x": x, "y": y},
             {"kind": "tokens_in", "src": vals, "y": y}]
    for spec in specs:
        assert _audit_one(spec, {}, [0, 2]) == [(spec["kind"], 0.0)]
    y.buf.tensor.view({torch.float16: torch.int16, torch.float32: torch.int32}[tdt])[2 * N * C + 7] += 1
    out.tensor.view(torch.int32)[2 * N * C + 3] += 1
    for spec in specs:
        with pytest.raises(AssertionError):
            _audit_one(spec, {}, [0, 2])


def test_channel_affine_bound_rejects_f16_storage_in_f32():
    g = torch.Generator().manual_seed(2)
    B, N, C = 2, 7, 24
    x = torch.randn(B, N, C, generator=g)
    sc, sh = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    y = _fma(x, sc, sh)
    spec = {"kind": "channel_affine", "x": _tok(B, N, C, L.PV_F32, x), "y": _tok(B, N, C, L.PV_F32, y),
            "scale": sc, "shift": sh}
    assert _audit_one(spec, {}, [0, 1])[0][1] <= 1.0
    spec["y"] = _tok(B, N, C, L.PV_F32, y.half().float())
    with pytest.raises(AssertionError):
        _audit_one(spec, {}, [0, 1])


def test_roi_align_reference_rejects_a_contracted_geometry():
    """RoIAlign as the audit checks it: the fp32 emulation of torchvision's geometry passes; the same geometry with
    `end * scale - start` and `start + ph * bin` contracted into FMAs takes another sample count for this box (one
    of test_gpu_input_matrix.py's contraction boxes) and fails."""
    import types
    g = torch.Generator().manual_seed(8)
    N, H, W, C = 2, 16, 16, 16
    geom = (3, 2, 1 / 12, 0)
    boxes = [(0, 1.0, 10.73066520690918, 40.0, 82.73066711425781), (1, 2.0, 3.0, 150.0, 120.0)]
    x = torch.randn(N, H, W, C, generator=g)
    xt = TRef(Buf(x.numel(), L.PV_F32), N, 1, H, W, C, Cp=C)
    xt.buf.tensor = x.reshape(-1).clone()
    rois = types.SimpleNamespace(tensor=torch.tensor(boxes, dtype=torch.float32))
    launched = {"roi_align_kernel<float>": 1}
    for contract in (False, True):
        y, _ = TS.roi_ref64(x, boxes, geom, emulate=True, contract=contract)
        yt = TRef(Buf(y.numel(), L.PV_F32), len(boxes), 1, 3, 2, C, Cp=C)
        yt.buf.tensor = y.reshape(-1).clone()
        spec = {"kind": "roi_align", "x": xt, "rois": rois, "y": yt, "geom": geom}
        if contract:
            with pytest.raises(AssertionError):
                _audit_one(spec, launched, [0])
        else:
            assert _audit_one(spec, launched, [0])[0][1] <= 1.0


def _mask_ref(m):
    import types
    return types.SimpleNamespace(tensor=m.to(torch.uint8), buf=None, B=m.shape[0], T=m.shape[1])


@pytest.mark.parametrize("divide_by_t", [False, True])
def test_masked_average_reference_rejects_a_division_by_t(divide_by_t):
    """fp32 masked average (sum of the valid steps in order, / the valid count, 1 when none) passes; the same sum
    divided by T fails."""
    x = torch.randn(5, 7, 16, generator=torch.Generator().manual_seed(4))
    m = torch.tensor(TS.MASKED_MASK, dtype=torch.bool)
    acc = torch.zeros(5, 16)
    for t in range(7):
        acc = acc + x[:, t] * m[:, t:t + 1]
    cnt = m.sum(1, keepdim=True).clamp_min(1).float()
    y = acc / (7.0 if divide_by_t else cnt)
    spec = {"kind": "masked_pool", "x": _tok(5, 7, 16, L.PV_F32, x), "mask": _mask_ref(m), "mode": L.MPOOL_AVG,
            "y": _tok(5, 1, 16, L.PV_F32, y)}
    clips = [0, 2, 4]
    if divide_by_t:
        with pytest.raises(AssertionError):
            _audit_one(spec, {"masked_pool_kernel<float,1>": 1}, clips)
    else:
        assert _audit_one(spec, {"masked_pool_kernel<float,1>": 1}, clips)[0][1] <= 1.0


def _lstm_kernel_f32(G, W, lengths, H, nd, swap_if=False):
    """fp32 LSTM recurrence in the kernel's order: z = G + h W^T, gates i, f, g, o, c = f c + i g, h = o tanh(c).
    swap_if: a wrong kernel that applies the input gate to the cell and the forget gate to the candidate."""
    B = G.shape[0]
    out = torch.zeros(B, nd * H)
    for b in range(B):
        n = int(lengths[b])
        for d in range(nd):
            h, c = torch.zeros(H), torch.zeros(H)
            for s in range(n):
                t = s if d == 0 else n - 1 - s
                z = G[b, t, d * 4 * H:(d + 1) * 4 * H]
                for j in range(H):
                    z = _fma(h[j], W[d, j], z)
                i, f, gg, o = z[:H].sigmoid(), z[H:2 * H].sigmoid(), z[2 * H:3 * H].tanh(), z[3 * H:].sigmoid()
                if swap_if:
                    i, f = f, i
                c = f * c + i * gg
                h = o * c.tanh()
            out[b, d * H:(d + 1) * H] = h
    return out


@pytest.mark.parametrize("swap_if", [False, True])
def test_lstm_bound_accepts_the_kernel_and_rejects_swapped_gates(swap_if):
    g = torch.Generator().manual_seed(6)
    B, T, H, nd = 5, 7, 24, 2
    G = torch.randn(B, T, nd * 4 * H, generator=g)
    W = torch.randn(nd, H, 4 * H, generator=g) * (0.5 / H ** 0.5)
    m = torch.tensor(TS.MASKED_MASK, dtype=torch.bool)
    y = _lstm_kernel_f32(G, W, m.sum(1).clamp(1, T), H, nd, swap_if=swap_if)
    spec = {"kind": "lstm", "g": _tok(B, T, nd * 4 * H, L.PV_F32, G), "mask": _mask_ref(m),
            "y": _tok(B, 1, nd * H, L.PV_F32, y), "w_hh_t": W, "hidden": H, "dirs": nd}
    launched = {"lstm_recurrence_kernel<float>": 1}
    if swap_if:
        with pytest.raises(AssertionError):
            _audit_one(spec, launched, [0, 2, 4])
    else:
        assert _audit_one(spec, launched, [0, 2, 4])[0][1] <= 1.0


def test_attention_weights_bound_accepts_the_kernel_and_rejects_a_missing_head_average():
    """pv_attention_weights in fp32: sum_h __expf(s - lse_h) / H from the attention launch's row log-sum-exp passes;
    the sum without the division by H fails."""
    g = torch.Generator().manual_seed(9)
    B, H, N, D = 3, 2, 40, 32
    q, k = (torch.randn(B, H, N, D, generator=g) for _ in range(2))
    m = torch.rand(B, N, generator=g) < 0.6
    m[2] = False
    scale = D ** -0.5
    s = torch.zeros(B, H, N, N)
    qs = q * scale
    for c in range(D):
        s = _fma(qs[..., c:c + 1], k[..., c].unsqueeze(2), s)
    s = s.masked_fill(~m[:, None, None, :], -math.inf)
    lse = torch.logsumexp(s, -1, keepdim=True)
    e = torch.where(torch.isneginf(lse), torch.zeros_like(s), torch.exp(s - lse))
    for div in (True, False):
        w = e.sum(1) / (H if div else 1)
        spec = {"kind": "attention_weights", "q": _tok(B, N, H * D, L.PV_F32, _rows(q)),
                "k": _tok(B, N, H * D, L.PV_F32, _rows(k)), "mask": _mask_ref(m), "lse": None,
                "w": Buf(w.numel(), L.PV_F32), "heads": H, "scale": scale}
        spec["w"].tensor = w.reshape(-1).clone()
        if div:
            assert _audit_one(spec, {"attention_weights_kernel<float>": 1}, [0, 1, 2])[0][1] <= 1.0
        else:
            with pytest.raises(AssertionError):
                _audit_one(spec, {"attention_weights_kernel<float>": 1}, [0, 1, 2])
