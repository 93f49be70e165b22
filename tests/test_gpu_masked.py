"""The masked multistream modules (models/masked_multistream.py), the fusion layers (layers/fusion.py), PositionalEncoding
and their kernels: the key-masked attention instances and the attention weights (csrc/pv_attention*.cu) and the masked
sequence ops (csrc/pv_masked.cu).

CPU: module trees against tests/golden/masked.pt (state_dict keys and repr, written by oracle/gen_golden_masked.py from
the real reference), the lowerings' launch lists and FLOP counts, the ReduceFusion classification, error types, the
routing of pv_attention_masked_fwd and the ledger of the masked instances.

GPU: every masked-attention instance against float64 with the launched instance asserted (a key tile with every key
masked, rows where only key 0 is valid, a row with no valid key), bitwise equality with pv_attention_fwd under an
all-valid mask, the weights kernel against float64, every golden case in f32 parity mode and in f16, attention_weights
after a nested forward, one plan replayed with two masks, caller tensors left unchanged, and the error paths.
"""
import ctypes as C
import os
import re

import pytest
import torch
import torch.nn as nn

from pytorchvideo_b200 import testing as TS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pytorchvideo_b200", "csrc")
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "masked.pt"), weights_only=False)

# f16 engine vs the reference's fp32 CPU forward, max |err| / max |ref| per case: about twice what was measured on an
# H100 80GB HBM3 at a 400 W power limit, which ranged from 2.8e-4 (pool_max, encoder_1) to 7.8e-4 (encoder_2).
MASKED_F16_BOUNDS = {"pool_max": 6e-4, "pool_avg": 1e-3, "pool_sum": 9e-4, "pool_avg_nomask": 9e-4, "pool_max_t1": 7e-4,
                     "default": 7e-4, "posenc": 9e-4, "mha": 1e-3, "mha_nomask": 9e-4, "mha_d32_t1": 7e-4,
                     "mha_d128": 9e-4, "chain": 1.4e-3, "encoder_1": 6e-4, "encoder_2": 1.6e-3, "encoder_nomask": 7e-4,
                     "lstm_uni": 7e-4, "lstm_bi": 9e-4, "lstm_bi_t1": 1.3e-3, "lstm_nomask": 9e-4,
                     "multipath_concat": 8e-4, "multipath_temporal_concat": 8e-4, "multipath_max": 1e-3,
                     "multipath_sum": 1.2e-3, "multipath_prod": 8e-4}


def _ns():
    return TS.masked_namespace()


def _lib():
    from pytorchvideo_b200 import _lib as L
    return L


def _lower(case, dtype="f16"):
    from pytorchvideo_b200.engine.lower import lower_only
    m = TS.build_masked_case(case, _ns())
    x, mask = TS.masked_case_inputs(case)
    ins, extra = TS.masked_engine_args(case, x, mask)
    return lower_only(m, ins, dtype=dtype, extra=extra)


@pytest.mark.parametrize("case", TS.MASKED_CASES)
def test_lowering_matches_reference_tree(case):
    """The reference's own module tree (launch list stored by oracle/gen_golden_masked.py) lowers as this package's."""
    assert [op["name"] for op in _lower(case)[0].meta] == GOLD[case]["ref_launches"]


# ---- CPU: module trees ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", TS.MASKED_CASES)
def test_module_tree_matches_reference(case):
    m = TS.build_masked_case(case, _ns(), seed=GOLD[case]["seed"])
    assert repr(m) == GOLD[case]["repr"]
    assert list(m.state_dict().keys()) == GOLD[case]["keys"]
    assert TS.state_checksum(m) == GOLD[case]["state_checksum"]
    x, _ = TS.masked_case_inputs(case)
    assert TS.tensor_checksum(x) == GOLD[case]["input_checksum"]


@pytest.mark.parametrize("case", TS.MASKED_CASES)
def test_oracle_matches_goldens(case):
    """oracle/masked_ref.py against the reference's outputs: bit-exact where it repeats the reference's own ops."""
    from oracle.masked_ref import masked_forward
    m = TS.build_masked_case(case, _ns(), seed=GOLD[case]["seed"])
    x, mask = TS.masked_case_inputs(case)
    ref = GOLD[case]["output"]
    y, w = masked_forward(m, x, mask)
    if case.startswith(("pool_", "default", "posenc")):
        assert torch.equal(y, ref)
    else:
        assert float((y - ref).abs().max()) <= 2e-6 * float(ref.abs().max())
    assert sorted(w) == sorted(GOLD[case]["weights"])
    for n, wr in GOLD[case]["weights"].items():
        assert float((w[n] - wr).abs().max()) <= 2e-6


def test_module_attributes():
    ns = _ns()
    lstm = ns.LSTM(16, 8, bidirectional=True)
    assert lstm.output_dim == 16 and lstm.bidirectional and lstm.lstm.batch_first
    assert sorted(k for k in lstm.state_dict()) == sorted(
        ["lstm.%s_l0%s" % (w, r) for w in ("weight_ih", "weight_hh", "bias_ih", "bias_hh") for r in ("", "_reverse")])
    assert ns.make_fusion_layer("concat", [8, 16]).output_dim == 24
    assert ns.make_fusion_layer("max", [8, 8]).output_dim == 8
    with pytest.raises(NotImplementedError):
        ns.make_fusion_layer("mean", [8, 8])
    pe = ns.PositionalEncoding(8, seq_len=4)
    assert tuple(pe.pe.shape) == (1, 4, 8) and float(pe.pe[0, 1, 0]) == pytest.approx(0.8414709848)


# ---- CPU: lowering ---------------------------------------------------------------------------------------------------
def _names(plan):
    return [m["name"] for m in plan.meta]


def test_lowering_chain_launch_list():
    plan, shape = _lower("chain")
    assert shape == (5, 64)
    assert _names(plan) == ["tokens_in", "0", "2.mask", "2._attention.in_proj", "2._attention.attention",
                            "2._attention.attention.weights", "2._attention.out_proj", "3", "4", "5", "output.to_tokens"]
    att = [m for m in plan.meta if m["kind"] == "attention"]
    assert len(att) == 1 and att[0]["flops"] == 4.0 * 5 * 2 * 7 * 7 * 32
    assert plan.attention_calls[-1]["masked"] and plan.attention_calls[-1]["D"] == 32


def test_lowering_encoder_launch_list_and_flops():
    for case, layers in (("encoder_1", 1), ("encoder_2", 2)):
        plan, shape = _lower(case)
        assert shape == (5, 64)
        per = ["self_attn.in_proj", "self_attn.attention", "self_attn.out_proj", "norm1", "linear1", "linear2", "norm2"]
        want = ["tokens_in", "TransposeTransformerEncoder.mask"] + [
            "TransposeTransformerEncoder.encoder.layers.%d.%s" % (i, n) for i in range(layers) for n in per]
        assert _names(plan)[:len(want)] == want
        lin1 = [m for m in plan.meta if m["name"].endswith("linear1")]
        assert [m["flops"] for m in lin1] == [2.0 * 5 * 7 * 2048 * 64] * layers
    plan, _ = _lower("encoder_nomask")
    assert not any(n.endswith(".mask") for n in _names(plan))


@pytest.mark.parametrize("fusion", TS.MASKED_FUSIONS)
def test_lowering_multipath(fusion):
    plan, shape = _lower("multipath_" + fusion)
    assert shape == ((5, 128) if fusion in ("concat", "temporal_concat") else (5, 64))
    names = _names(plan)
    assert "multipathway_blocks.0.0.mask" in names and "multipathway_blocks.1.1.lstm.recurrence" in names
    stream_lanes = {m["lane"] for m in plan.meta if m["name"].startswith("multipathway_blocks.1")}
    assert stream_lanes == {1}
    if fusion in ("concat", "temporal_concat"):
        assert "multipathway_fusion" not in names      # the streams write channel slices of one buffer
    else:
        assert "multipathway_fusion" in names


def test_lowering_lstm_launch_list_and_flops():
    plan, shape = _lower("lstm_bi")
    assert shape == (5, 64)
    assert _names(plan) == ["tokens_in", "LSTM.lstm.input_proj", "LSTM.lstm.recurrence", "output.to_tokens"]
    proj, rec = plan.meta[1], plan.meta[2]
    assert proj["flops"] == 2.0 * 5 * 7 * (2 * 4 * 32) * 64          # both directions in one GEMM
    assert rec["flops"] == 2.0 * 2 * 5 * 7 * 4 * 32 * 32
    plan, shape = _lower("lstm_uni")
    assert shape == (5, 48) and plan.meta[1]["flops"] == 2.0 * 5 * 7 * (4 * 48) * 64


def test_reference_style_layer_lowerings():
    """Plain nn.LayerNorm / nn.Linear on token tensors lower; Dropout is the identity."""
    from pytorchvideo_b200.engine.lower import lower_only
    seq = nn.Sequential(nn.Linear(64, 32), nn.Dropout(0.1), nn.LayerNorm(32))
    plan, shape = lower_only(seq, torch.randn(2, 5, 64))
    assert shape == (2, 5, 32) and _names(plan) == ["tokens_in", ".0", ".2", "output.to_tokens"]


def _fusion_ref(method, ins):
    if method == "concat":
        return torch.cat(ins, dim=-1)
    if method == "temporal_concat":
        return torch.cat(ins, dim=1)
    return {"max": lambda x: torch.max(x, dim=0).values, "sum": lambda x: torch.sum(x, dim=0),
            "prod": lambda x: torch.prod(x, dim=0)}[method](torch.stack(ins))


FUSION_ROOT_SHAPES = [(5, 64), (5, 3, 64)]


@pytest.mark.parametrize("method", TS.MASKED_FUSIONS)
@pytest.mark.parametrize("shape", FUSION_ROOT_SHAPES)
def test_fusion_layer_alone_lowers_to_torch_shape(method, shape):
    """A fusion layer called on its own keeps the rank of its inputs: (batch, feature) inputs give a 2-D result."""
    from pytorchvideo_b200.engine.lower import lower_only
    ins = [torch.randn(*shape), torch.randn(*shape)]
    assert lower_only(_ns().make_fusion_layer(method, [64, 64]), ins)[1] == tuple(_fusion_ref(method, ins).shape)


def test_reduce_fusion_classification():
    from pytorchvideo_b200.engine.lower import reduce_fusion_op
    L = _lib()
    ns = _ns()
    assert reduce_fusion_op(ns.make_fusion_layer("max", [8, 8]).reduce_fn) == L.REDUCE_MAX
    assert reduce_fusion_op(ns.make_fusion_layer("sum", [8, 8]).reduce_fn) == L.REDUCE_SUM
    assert reduce_fusion_op(ns.make_fusion_layer("prod", [8, 8]).reduce_fn) == L.REDUCE_PROD
    for fn in (lambda x: torch.mean(x, dim=0), lambda x: torch.min(x, dim=0).values, lambda x: x[0], lambda x: "no"):
        with pytest.raises(NotImplementedError):
            reduce_fusion_op(fn)


def test_unsupported_configurations_raise_not_implemented():
    from pytorchvideo_b200.engine.lower import lower_only
    ns = _ns()
    x, mask = torch.randn(2, 4, 48), torch.ones(2, 4, dtype=torch.bool)
    with pytest.raises(NotImplementedError, match="head dim 48"):
        lower_only(ns.TransposeMultiheadAttention(48, 1), [x, mask], extra=(("masks", False, True),))
    with pytest.raises(NotImplementedError, match="head dim 256"):
        lower_only(ns.TransposeMultiheadAttention(256, 1), [torch.randn(2, 4, 256), mask], extra=(("masks", False, True),))
    with pytest.raises(NotImplementedError, match="hidden_dim=513"):
        lower_only(ns.LSTM(48, 513), [x, mask], extra=(("masks", False, True),))
    with pytest.raises(NotImplementedError, match="hidden_dim=600"):
        lower_only(ns.MaskedSequential(ns.LSTM(48, 600, bidirectional=True)), [x, mask], extra=(("masks", False, True),))


def _route_masked(D, dtype="f16", q=0x10000):
    L = _lib()
    d = L.AttentionDesc()
    d.dtype, d.B, d.H, d.Nq, d.Nk, d.D = (L.PV_F16 if dtype == "f16" else L.PV_F32), 2, 2, 9, 9, D
    rs = 3 * 2 * D
    d.q_row_stride = d.k_row_stride = d.v_row_stride = rs
    d.q_batch_stride = d.k_batch_stride = d.v_batch_stride = 9 * rs
    d.o_row_stride, d.o_batch_stride, d.scale = 2 * D, 18 * D, D ** -0.5
    return L.load().pv_attention_kernel_for(C.byref(d), q, 0x20000, 0x30000, 0x40000)


def test_masked_routing():
    """pv_attention_masked_fwd takes the route pv_attention_kernel_for gives: wgmma for 32 / 64 / 96, mma for 128, the
    CUDA-core kernel for f32 or misaligned operands."""
    L = _lib()
    for D, k in ((32, L.ATTN_WGMMA), (64, L.ATTN_WGMMA), (96, L.ATTN_WGMMA), (128, L.ATTN_MMA)):
        assert _route_masked(D) == k
        assert _route_masked(D, "f32") == L.ATTN_SIMT
        assert _route_masked(D, q=0x10008) == L.ATTN_SIMT


def masked_instances():
    def src(f):
        return open(os.path.join(CSRC, f)).read()
    out = set()
    for dd in re.findall(r"PV_AWM\((\d+)\)", src("pv_attention_wgmma.cu")):
        out.add("attention_wgmma_masked_kernel<%s>" % dd)
    for dd in re.findall(r"PV_AMM\((\d+)\)", src("pv_attention_mma.cu")):
        out.add("attention_mma_masked_kernel<%s>" % dd)
    for dd in re.findall(r"PV_ATTM\((\d+)\)", src("pv_attention.cu")):
        out.update({"attention_masked_kernel<__half,%s>" % dd, "attention_masked_kernel<float,%s>" % dd})
    for t in re.findall(r'"(lstm_\w+_kernel(?:<\w+>)?)"', src("pv_lstm.cu")):
        out.add(t)
    return out


# (instance, dtype, D, alignment) rows of the GPU matrix below
MASKED_ROWS = ([("attention_wgmma_masked_kernel<%d>" % D, "f16", D, True) for D in (32, 64, 96)] +
               [("attention_mma_masked_kernel<128>", "f16", 128, True)] +
               [("attention_masked_kernel<__half,%d>" % D, "f16", D, False) for D in (32, 64, 96, 128)] +
               [("attention_masked_kernel<float,%d>" % D, "f32", D, True) for D in (32, 64, 96, 128)])


# (instance, dtype) rows of the LSTM matrix below
LSTM_ROWS = [("lstm_cluster_kernel", "f16"), ("lstm_recurrence_kernel<float>", "f32")]
# (B, T, H, directions): cluster sizes 1 (H = 32 / 64 / 96), 4 (256, 64 units per CTA), 12 (384) and 16 (512, two
# clusters per direction at B = 33)
LSTM_SHAPES = [(19, 37, 64, 2), (5, 512, 32, 1), (9, 1, 512, 2), (33, 20, 512, 2), (3, 9, 96, 1), (40, 11, 256, 2),
               (7, 13, 384, 2)]


def test_masked_instance_ledger():
    compiled = masked_instances()
    assert len(compiled) == 15
    # lstm_recurrence_kernel<__half>: f16 hidden sizes the cluster kernel cannot split (H = 300 below)
    assert compiled == {r[0] for r in MASKED_ROWS} | {r[0] for r in LSTM_ROWS} | {"lstm_recurrence_kernel<__half>"}


# ---- GPU: kernels --------------------------------------------------------------------------------------------------
def _mask_pattern(B, Nk, seed=3):
    g = torch.Generator().manual_seed(seed)
    m = torch.rand(B, Nk, generator=g) < 0.6
    m[0] = False
    m[0, 0] = True                      # only key 0 valid
    if Nk > 64:
        m[1, :] = True
        m[1, 64:128] = False            # a 64-key tile with every key masked
    m[2 % B] = False                    # no valid key at all
    return m


def _attention_case(dtype, D, aligned, B=3, H=2, N=150, seed=0):
    """q / k / v as channel slices of one qkv buffer, as the in-projection leaves them."""
    g = torch.Generator().manual_seed(seed)
    tdt = torch.float16 if dtype == "f16" else torch.float32
    W = 3 * H * D + (0 if aligned else 4)
    qkv = (torch.randn(B, N, W, generator=g) * 0.7).to(tdt).cuda()
    o = torch.zeros(B, N, H * D, dtype=tdt, device="cuda")
    return qkv, o, W


def _desc(dtype, B, H, N, D, W):
    L = _lib()
    d = L.AttentionDesc()
    d.dtype, d.B, d.H, d.Nq, d.Nk, d.D = (L.PV_F16 if dtype == "f16" else L.PV_F32), B, H, N, N, D
    d.q_row_stride = d.k_row_stride = d.v_row_stride = W
    d.q_batch_stride = d.k_batch_stride = d.v_batch_stride = N * W
    d.o_row_stride, d.o_batch_stride = H * D, N * H * D
    d.scale = D ** -0.5
    return d


def _ref64(qkv, B, H, N, D, mask):
    x = qkv.double().cpu()
    q, k, v = (x[..., i * H * D:(i + 1) * H * D].reshape(B, N, H, D).transpose(1, 2) for i in range(3))
    o, ao = TS.attn_ref64(q, k, v, D ** -0.5, False, mask=mask)
    p = TS.attn_probs64(q, k, D ** -0.5, mask)
    return o.transpose(1, 2).reshape(B, N, H * D), ao.transpose(1, 2).reshape(B, N, H * D), p


@pytest.mark.gpu
@pytest.mark.parametrize("row", MASKED_ROWS, ids=[r[0] + ("" if r[3] else "-unaligned") for r in MASKED_ROWS])
def test_gpu_masked_attention_against_f64(row):
    inst, dtype, D, aligned = row
    L = _lib()
    B, H, N = 3, 2, 150
    qkv, o, W = _attention_case(dtype, D, aligned, B, H, N)
    mask = _mask_pattern(B, N)
    mk = mask.to(torch.uint8).cuda()
    lse = torch.full((B, H, N), 7.0, device="cuda")
    d = _desc(dtype, B, H, N, D, W)
    esz = qkv.element_size()
    base = qkv.data_ptr()

    def run():
        L.check(L.load().pv_attention_masked_fwd(C.byref(d), base, base + H * D * esz, base + 2 * H * D * esz,
                                                 o.data_ptr(), mk.data_ptr(), lse.data_ptr(), None), "masked")
        torch.cuda.synchronize()
    _, launched = TS.launched_kernels(run)
    assert launched == {inst: 1}
    ref, aref, p = _ref64(qkv, B, H, N, D, mask)
    if dtype == "f16":
        TS.assert_close_to_f64(o, ref, aref, N, acc_eps=2.0 ** -9, what=inst)
    else:
        assert float((o.double().cpu() - ref).abs().max()) <= 1e-5 * (1 + float(aref.max()))
    assert bool((o[2 % B].float() == 0).all())                          # no valid key: o = 0
    assert bool(torch.isneginf(lse[2 % B]).all()) and bool(torch.isfinite(lse[:2]).all())
    # weights from the lse
    w = torch.empty(B, N, N, device="cuda")
    L.check(L.load().pv_attention_weights(C.byref(d), base, base + H * D * esz, mk.data_ptr(), lse.data_ptr(),
                                          w.data_ptr(), None), "weights")
    torch.cuda.synchronize()
    wref = p.mean(1)
    assert float((w.double().cpu() - wref).abs().max()) <= (2e-3 if dtype == "f16" else 1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,D,aligned", [("f16", 64, True), ("f16", 128, True), ("f16", 32, False), ("f32", 96, True)])
def test_gpu_all_valid_mask_is_bitwise_unmasked(dtype, D, aligned):
    L = _lib()
    B, H, N = 2, 2, 130
    qkv, o, W = _attention_case(dtype, D, aligned, B, H, N, seed=4)
    o2 = torch.zeros_like(o)
    mk = torch.ones(B, N, dtype=torch.uint8, device="cuda")
    d = _desc(dtype, B, H, N, D, W)
    esz = qkv.element_size()
    base = qkv.data_ptr()
    ptrs = (base, base + H * D * esz, base + 2 * H * D * esz)
    L.check(L.load().pv_attention_fwd(C.byref(d), *ptrs, o.data_ptr(), None), "fwd")
    L.check(L.load().pv_attention_masked_fwd(C.byref(d), *ptrs, o2.data_ptr(), mk.data_ptr(), None, None), "masked")
    torch.cuda.synchronize()
    assert torch.equal(o, o2)


@pytest.mark.gpu
@pytest.mark.parametrize("row", LSTM_ROWS, ids=[r[0] for r in LSTM_ROWS])
@pytest.mark.parametrize("B,T,H,nd", LSTM_SHAPES)
def test_gpu_lstm_recurrence_against_f64(row, B, T, H, nd):
    """Ragged and non-prefix masks, rows with no valid step (length clamped to 1), T up to 512, batches over more
    than one CTA / cluster, every cluster size; the length is a count of valid steps.  The f16 kernel multiplies f16
    W_hh and f16 h on the tensor cores: the reference takes both rounded to f16."""
    inst, dtype = row
    _lstm_check(inst, dtype, B, T, H, nd)


@pytest.mark.gpu
def test_gpu_lstm_f16_without_cluster_split():
    _lstm_check("lstm_recurrence_kernel<__half>", "f16", 4, 6, 300, 2)


def _lstm_check(inst, dtype, B, T, H, nd):
    L = _lib()
    g = torch.Generator().manual_seed(B * T + H)
    tdt = torch.float16 if dtype == "f16" else torch.float32
    G = (torch.randn(B, T, nd * 4 * H, generator=g)).to(tdt).cuda()
    W = (torch.randn(nd, H, 4 * H, generator=g) * (0.5 / H ** 0.5)).cuda()
    mask = torch.rand(B, T, generator=g) < 0.5
    mask[0] = False
    mask[1 % B] = True
    lengths = mask.sum(1).clamp(1, T)
    mk = mask.to(torch.uint8).cuda()
    y = torch.full((B, nd * H + 8), 9.0, dtype=tdt, device="cuda")

    def run():
        L.check(L.load().pv_lstm_recurrence(G.data_ptr(), L.PV_F16 if dtype == "f16" else L.PV_F32, nd * 4 * H,
                                            W.data_ptr(), mk.data_ptr(), B, T, H, nd, y.data_ptr(), nd * H + 8, None),
                "lstm")
        torch.cuda.synchronize()
    _, launched = TS.launched_kernels(run)
    assert launched == {inst: 1}
    ref, _ = TS.lstm_ref64(G, W.half() if inst == "lstm_cluster_kernel" else W, lengths, H, nd,
                           h16=inst == "lstm_cluster_kernel")
    err = float((y[:, :nd * H].double().cpu() - ref).abs().max())
    assert err <= (2e-3 if dtype == "f16" else 2e-5), err
    assert bool((y[:, nd * H:] == 9.0).all())                       # nothing written past the row


@pytest.mark.gpu
@pytest.mark.parametrize("method", TS.MASKED_FUSIONS)
@pytest.mark.parametrize("shape", FUSION_ROOT_SHAPES)
def test_gpu_fusion_layer_alone(method, shape):
    from pytorchvideo_b200 import config
    g = torch.Generator().manual_seed(11)
    ins = [torch.randn(*shape, generator=g), torch.randn(*shape, generator=g)]
    ref = _fusion_ref(method, ins)
    f = _ns().make_fusion_layer(method, [64, 64]).cuda().eval()
    old = config.get_precision()
    config.set_precision("f32")
    try:
        with torch.no_grad():
            y = f([t.cuda() for t in ins])
    finally:
        config.set_precision(old)
    assert tuple(y.shape) == tuple(ref.shape)
    assert float((y.cpu() - ref).abs().max()) <= 1e-6 * float(ref.abs().max())


# ---- GPU: modules against the goldens ------------------------------------------------------------------------------
def _run_case(case, precision):
    from pytorchvideo_b200 import config
    m = TS.build_masked_case(case, _ns(), seed=GOLD[case]["seed"]).cuda()
    x, mask = TS.masked_case_inputs(case)
    x, mask = x.cuda(), (mask.cuda() if mask is not None else None)
    old = config.get_precision()
    config.set_precision(precision)
    try:
        with torch.no_grad():
            y = TS.masked_call(m, x, mask)
    finally:
        config.set_precision(old)
    return m, y


@pytest.mark.gpu
@pytest.mark.parametrize("case", TS.MASKED_CASES)
def test_gpu_golden_f32_parity(case):
    m, y = _run_case(case, "f32")
    ref = GOLD[case]["output"]
    scale = float(ref.abs().max())
    err = (y.cpu() - ref).abs()
    assert bool((err <= 1e-3 * ref.abs() + 1e-4 * scale).all()), (case, float(err.max()))
    for n, w in GOLD[case]["weights"].items():
        got = m.get_submodule(n).attention_weights if n else m.attention_weights
        assert float((got.cpu() - w).abs().max()) <= 1e-4, (case, n)


@pytest.mark.gpu
@pytest.mark.parametrize("case", TS.MASKED_CASES)
def test_gpu_golden_f16(case):
    m, y = _run_case(case, "f16")
    ref = GOLD[case]["output"]
    rel = float((y.cpu() - ref).abs().max()) / float(ref.abs().max())
    print("MASKED_F16 %s %.3e" % (case, rel))
    assert rel <= MASKED_F16_BOUNDS[case], (case, rel)


@pytest.mark.gpu
def test_gpu_attention_weights_after_nested_forward():
    m, _ = _run_case("chain", "f32")
    w = m[2].attention_weights
    assert w is not None and w.dtype == torch.float32 and tuple(w.shape) == (5, 7, 7)
    assert float((w.cpu() - GOLD["chain"]["weights"]["2"]).abs().max()) <= 1e-4


@pytest.mark.gpu
def test_gpu_one_plan_two_masks():
    """The mask is plan data: one compiled plan (one CUDA graph) serves two masks of the same shape."""
    ns = _ns()
    m = TS.build_masked_case("chain", ns).cuda()
    x, mask = TS.masked_case_inputs("chain")
    x = x.cuda()
    other = torch.ones_like(mask)
    other[:, 3:] = False
    outs = []
    for mk in (mask, other, mask):
        with torch.no_grad():
            outs.append(m(input=x, mask=mk.cuda()))
    assert len(m.__dict__["_pv_cache"]) == 1
    assert torch.equal(outs[0], outs[2]) and not torch.equal(outs[0], outs[1])
    # the second mask against a fresh module, compiled for that mask alone (same default precision)
    m2 = TS.build_masked_case("chain", ns).cuda()
    with torch.no_grad():
        fresh = m2(input=x, mask=other.cuda())
    assert torch.equal(fresh, outs[1])


@pytest.mark.gpu
def test_gpu_caller_tensors_unchanged():
    for case in ("pool_max", "chain", "encoder_1", "multipath_concat"):
        m = TS.build_masked_case(case, _ns()).cuda()
        x, mask = TS.masked_case_inputs(case)
        x, mask = x.cuda(), mask.cuda()
        x0, m0 = x.clone(), mask.clone()
        with torch.no_grad():
            TS.masked_call(m, x, mask)
        assert torch.equal(x, x0) and torch.equal(mask, m0), case


@pytest.mark.gpu
def test_gpu_error_paths():
    ns = _ns()
    m = TS.build_masked_case("chain", ns)
    x, mask = TS.masked_case_inputs("chain")
    with pytest.raises(RuntimeError):
        m(input=x, mask=mask)                                  # CPU tensors
    m = m.cuda()
    with pytest.raises(RuntimeError):
        m(input=x.cuda(), mask=mask.cuda().float())            # a non-bool mask
    m.train()
    with pytest.raises(RuntimeError):
        m(input=x.cuda(), mask=mask.cuda())
    mp = TS.build_masked_case("multipath_sum", ns).cuda()
    mp.multipathway_fusion = None
    with pytest.raises(RuntimeError, match="multipathway_fusion"):
        mp([(x.cuda(), mask.cuda()), (x.cuda(), mask.cuda())])
    with pytest.raises(NotImplementedError):
        ns.LSTM(64, 600).cuda().eval()(x.cuda(), mask.cuda())
