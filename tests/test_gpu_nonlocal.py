"""The Non-local block (layers/nonlocal_net.py) and its attention core (csrc/pv_attention_wide.cu).

CPU: the routing of pv_attention_kernel_for with the ``normalize`` field, the lowering of NonLocal (launch list, fused
GEMMs, the attention problem, conv_out with the residual, error types), the instance ledger of the new kernels and
the oracle against tests/golden/nonlocal.pt (written by oracle/gen_golden_nonlocal.py from the real reference).

GPU: every instance x mode of the wide kernels against float64 (testing.assert_close_to_f64) with the launched
instance asserted, q / k / v read as channel slices of a theta|phi|g or a phi|g buffer; the late-maximum underflow
case; a large-magnitude linear-mode case; bitwise batch invariance.  Layer cases against the goldens in f16 and in
f32 parity mode, the transmute_model route, and i3d_r50 with the I3D-NLN layout of Non-local blocks.
"""
import ctypes as C
import os
import re

import pytest
import torch
import torch.nn as nn

from oracle.nonlocal_ref import nonlocal_forward
from pytorchvideo_b200 import testing as TS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pytorchvideo_b200", "csrc")
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "nonlocal.pt"), weights_only=False)


def _lib():
    from pytorchvideo_b200 import _lib as L
    return L


def _desc(dtype, B, Nq, Nk, D, q_rs, kv_rs, q_bs, kv_bs, o_rs, o_bs, normalize=0, resid=0, scale=None):
    L = _lib()
    d = L.AttentionDesc()
    d.dtype, d.B, d.H, d.Nq, d.Nk, d.D = dtype, B, 1, Nq, Nk, D
    d.q_row_stride, d.k_row_stride, d.v_row_stride, d.o_row_stride = q_rs, kv_rs, kv_rs, o_rs
    d.q_batch_stride, d.k_batch_stride, d.v_batch_stride, d.o_batch_stride = q_bs, kv_bs, kv_bs, o_bs
    d.scale = D ** -0.5 if scale is None else scale
    d.add_q_residual, d.normalize = resid, normalize
    return d


# ---- CPU: routing ----------------------------------------------------------------------------------------------------
def _route(D, dtype="f16", normalize=0, resid=0, q=0x10000, k=0x20000, v=0x30000, o=0x40000, rs_pad=0, H=1):
    L = _lib()
    N = 51
    d = _desc(L.PV_F16 if dtype == "f16" else L.PV_F32, 2, N, N, D, 3 * H * D + rs_pad, 3 * H * D + rs_pad,
              N * (3 * H * D + rs_pad), N * (3 * H * D + rs_pad), H * D, N * H * D, normalize, resid)
    d.H = H
    return L.load().pv_attention_kernel_for(C.byref(d), q, k, v, o)


def test_routing_wide_heads_and_linear_mode():
    L = _lib()
    for D in (256, 512):
        assert _route(D) == L.ATTN_WIDE
        assert _route(D, normalize=1) == L.ATTN_WIDE
        assert _route(D, dtype="f32") == L.ATTN_SIMT
        assert _route(D, dtype="f32", normalize=1) == L.ATTN_SIMT
        assert _route(D, q=0x10008) == L.ATTN_SIMT          # misaligned pointer
        assert _route(D, rs_pad=4) == L.ATTN_SIMT           # row stride not a multiple of 8 elements
        assert _route(D, o=0x40002) == L.ATTN_SIMT
        assert _route(D, resid=1) == L.ATTN_WIDE
    for D in (64, 128):
        assert _route(D, normalize=1) == L.ATTN_WIDE
        assert _route(D, normalize=1, dtype="f32") == L.ATTN_SIMT
        assert _route(D, normalize=1, k=0x20002) == L.ATTN_SIMT
    for D in (32, 96, 48, 1024, 768):
        assert _route(D, normalize=1) == -3                 # PV_ERR_UNSUPPORTED
    for D in (48, 1024, 384):
        assert _route(D) == -3
    assert _route(256, normalize=1, resid=1) == -1          # PV_ERR_INVALID: the linear mode takes no q residual
    assert _route(64, normalize=1, resid=1) == -1
    assert _route(256, normalize=2) == -1


def test_routing_with_zero_normalize_is_unchanged():
    """A zeroed ``normalize`` (every in-tree descriptor) routes the MViT head dims exactly as before."""
    L = _lib()
    for H in (1, 2):
        for D in (32, 64, 96):
            assert _route(D, H=H) == L.ATTN_WGMMA
            assert _route(D, H=H, dtype="f32") == L.ATTN_SIMT
            assert _route(D, H=H, q=0x10008) == L.ATTN_SIMT
        assert _route(128, H=H) == L.ATTN_MMA
        assert _route(128, H=H, o=0x40001) == L.ATTN_SIMT
    assert C.sizeof(L.AttentionDesc) == 104


# ---- CPU: lowering ---------------------------------------------------------------------------------------------------
def _nl(**kw):
    from pytorchvideo_b200.layers.nonlocal_net import create_nonlocal
    return create_nonlocal(**kw).eval()


def _lower(m, shape, dtype="f16"):
    from pytorchvideo_b200.engine.lower import lower_only
    return lower_only(m, torch.empty(shape), dtype=dtype)


@pytest.mark.parametrize("dtype", ["f16", "f32"])
def test_lower_nonlocal_with_pool(dtype):
    """I3D-NLN res3 at 8x224^2: 4x28x28 = 3136 queries, 784 keys after the (1,2,2) pool, D = 256."""
    plan, shape = _lower(_nl(dim_in=512, dim_inner=256, pool_size=(1, 2, 2)), (2, 512, 4, 28, 28), dtype)
    assert tuple(shape) == (2, 512, 4, 28, 28)
    names = [mm["name"] for mm in plan.meta]
    assert names == ["ncdhw_to_ndhwc", "nonlocal.conv_theta", "nonlocal.pool", "nonlocal.conv_phi_g", "nonlocal.attention",
                     "nonlocal.conv_out", "output.to_ncdhw"], names
    (a,) = plan.attention_calls
    assert (a["B"], a["H"], a["Nq"], a["Nk"], a["D"], a["normalize"], a["add_q_residual"]) == (2, 1, 3136, 784, 256, 0, 0)
    assert abs(a["scale"] - 256 ** -0.5) < 1e-7
    assert plan.meta[4]["flops"] == 4.0 * 2 * 3136 * 784 * 256
    # conv_out reads the attention output and x (the fused identity residual)
    reads = plan.op_io[5][0]
    assert len(reads) == 2 and reads[1].C == 512 and reads[0].C == 256
    # theta: one GEMM of 256 channels on x; phi|g: one GEMM of 512 channels on the pooled x
    assert plan.meta[1]["flops"] == 2.0 * 2 * 3136 * 256 * 512
    assert plan.meta[3]["flops"] == 2.0 * 2 * 784 * 512 * 512


def test_lower_nonlocal_without_pool_dot_product():
    plan, _ = _lower(_nl(dim_in=1024, dim_inner=512, pool_size=None, instantiation="dot_product"), (1, 1024, 2, 14, 14))
    names = [mm["name"] for mm in plan.meta]
    assert names == ["ncdhw_to_ndhwc", "nonlocal.conv_theta_phi_g", "nonlocal.attention", "nonlocal.conv_out",
                     "output.to_ncdhw"], names
    assert plan.meta[1]["flops"] == 2.0 * 392 * 1536 * 1024
    (a,) = plan.attention_calls
    assert (a["Nq"], a["Nk"], a["D"], a["normalize"], a["scale"]) == (392, 392, 512, 1, 1.0)


def test_lower_nonlocal_ragged_pool_and_i3d_res4():
    plan, _ = _lower(_nl(dim_in=256, dim_inner=128, pool_size=(1, 2, 2)), (1, 256, 3, 7, 9))
    (a,) = plan.attention_calls
    assert (a["Nq"], a["Nk"], a["D"]) == (3 * 7 * 9, 3 * 3 * 4, 128)
    plan, _ = _lower(_nl(dim_in=1024, dim_inner=512, pool_size=(1, 2, 2)), (8, 1024, 4, 14, 14))
    (a,) = plan.attention_calls
    assert (a["B"], a["Nq"], a["Nk"], a["D"]) == (8, 784, 196, 512)


def test_lower_nonlocal_errors():
    from pytorchvideo_b200.layers.nonlocal_net import NonLocal
    x = (1, 64, 2, 8, 8)
    with pytest.raises(NotImplementedError):                 # dim_inner without a kernel
        _lower(_nl(dim_in=64, dim_inner=48), x)
    with pytest.raises(NotImplementedError):                 # the linear mode has no 32-wide kernel
        _lower(_nl(dim_in=64, dim_inner=32, instantiation="dot_product"), x)
    with pytest.raises(NotImplementedError):
        _lower(_nl(dim_in=64, dim_inner=1024), x)
    m = _nl(dim_in=64, dim_inner=64)
    m.conv_theta = nn.Conv3d(64, 64, kernel_size=3, padding=1)
    with pytest.raises(NotImplementedError):
        _lower(m, x)
    m = _nl(dim_in=64, dim_inner=64)
    m.conv_g = nn.Conv3d(64, 64, kernel_size=1, stride=(1, 2, 2))
    with pytest.raises(NotImplementedError):
        _lower(m, x)
    m = _nl(dim_in=64, dim_inner=64)
    m.conv_phi = nn.Conv3d(64, 64, kernel_size=1, groups=2)
    with pytest.raises(NotImplementedError):
        _lower(m, x)
    m = NonLocal(conv_theta=nn.Conv3d(64, 64, 1), conv_phi=nn.Conv3d(64, 64, 1), conv_g=nn.Conv3d(64, 64, 1),
                 conv_out=nn.Conv3d(64, 64, 1), norm=nn.GroupNorm(4, 64), instantiation="softmax").eval()
    with pytest.raises(NotImplementedError):
        _lower(m, x)
    with pytest.raises(RuntimeError):                        # wrong channel count
        _lower(_nl(dim_in=64, dim_inner=64), (1, 32, 2, 8, 8))
    with pytest.raises(AssertionError):
        NonLocal(conv_theta=nn.Conv3d(64, 32, 1), conv_phi=nn.Conv3d(64, 64, 1), conv_g=nn.Conv3d(64, 64, 1),
                 conv_out=nn.Conv3d(64, 64, 1))
    with pytest.raises(AssertionError):
        _nl(dim_in=64, dim_inner=64, instantiation="gaussian")


def test_create_nonlocal_structure():
    m = _nl(dim_in=64, dim_inner=32)
    assert m.pool is None and m.instantiation == "softmax" and isinstance(m.norm, nn.BatchNorm3d)
    m = _nl(dim_in=64, dim_inner=32, pool_size=(1, 2, 2), norm=None, instantiation="dot_product")
    assert isinstance(m.pool, nn.MaxPool3d) and m.norm is None
    assert list(m.state_dict().keys())[:2] == ["conv_theta.weight", "conv_theta.bias"]
    import pytorchvideo_b200.layers as layers
    assert not hasattr(layers, "NonLocal")                  # like the reference, not exported from layers


# ---- CPU: oracle vs the reference's goldens --------------------------------------------------------------------------
@pytest.mark.parametrize("case", sorted(TS.NONLOCAL_CASES))
def test_oracle_matches_reference_golden(case):
    from pytorchvideo_b200.layers.nonlocal_net import create_nonlocal
    m, x = TS.build_nonlocal_case(case, create_nonlocal, seed=GOLD[case]["seed"])
    g = GOLD[case]
    assert abs(TS.state_checksum(m) - g["state_checksum"]) <= 1e-6 * abs(g["state_checksum"])
    assert TS.tensor_checksum(x) == pytest.approx(g["input_checksum"], rel=1e-9)
    ref = g["output"]
    out = nonlocal_forward(m, x)
    assert out.shape == ref.shape
    assert float((out - ref).abs().max()) <= 1e-5 * max(1.0, float(ref.abs().max()))


# ---- GPU kernel rows -------------------------------------------------------------------------------------------------
WIDE_NQ_NK = [(1, 1), (63, 64), (64, 65), (65, 63), (196, 196), (784, 196), (3136, 784), (64, 3136), (1, 784)]
SIMT_NQ_NK = [(1, 1), (65, 63), (196, 784), (3136, 64)]


def _wide_rows():
    rows = []
    for D, dout, modes in ((64, 64, (1,)), (128, 128, (1,)), (256, 256, (0, 1)), (512, 256, (0, 1))):
        for mode in modes:
            for i, (nq, nk) in enumerate(WIDE_NQ_NK):
                rows.append(("attention_wide_kernel<%d,%d>" % (D, dout), "f16", D, mode, nq, nk, 1 + 2 * (i % 2)))
    for D, modes in ((64, (1,)), (128, (1,)), (256, (0, 1)), (512, (0, 1))):
        for mode in modes:
            for i, (nq, nk) in enumerate(SIMT_NQ_NK):
                rows.append(("attention_wide_simt_kernel<float,%d>" % D, "f32", D, mode, nq, nk, 1 + 2 * (i % 2)))
                rows.append(("attention_wide_simt_kernel<__half,%d>" % D, "unaligned", D, mode, nq, nk,
                             3 - 2 * (i % 2)))
    return rows


WIDE_ROWS = _wide_rows()


def test_instance_ledger_covers_every_wide_instance():
    src = open(os.path.join(CSRC, "pv_attention_wide.cu")).read()
    compiled = {"attention_wide_kernel<%s,%s>" % (dd, do) for dd, do, _, _ in
                re.findall(r"PV_AWIDE\((\d+), (\d+), (\d+), (\d+)\)", src)}
    for dd in re.findall(r"PV_AWS\((\d+)\)", src):
        compiled |= {"attention_wide_simt_kernel<__half,%s>" % dd, "attention_wide_simt_kernel<float,%s>" % dd}
    assert len(compiled) == 12
    assert compiled == {r[0] for r in WIDE_ROWS}
    assert '"attention_wide_kernel<" #DD "," #DO ">"' in src


def _ref64(q, k, v, scale, normalize, resid=False):
    """q [B,Nq,D], k / v [B,Nk,D] on the f16 grid -> (ref64, absref64)."""
    return TS.attn_ref64(q, k, v, scale, resid, normalize)


ACC_EPS_ATTN = 2.0 ** -9       # P is rounded to f16 before P.V (tests/test_gpu_kernel_matrix.py, same bound)


def _dev():
    return torch.device("cuda:0")


def _run_attention(q, k, v, scale, normalize, mode, layout="slices", resid=False):
    """pv_attention_fwd with q / k / v as channel slices: with Nq == Nk of ONE theta|phi|g buffer [B][N][3D] (the
    un-pooled Non-local block), else q from a theta buffer and k / v from a phi|g buffer [B][Nk][2D] (pooled).  mode:
    f16, f32, or unaligned (f16 storage with o 2 bytes off the 4-byte alignment the tensor-core kernels store with: the
    CUDA-core kernel)."""
    L = _lib()
    B, Nq, D = q.shape
    Nk = k.shape[1]
    tdt = torch.float32 if mode == "f32" else torch.float16
    dt = L.PV_F32 if mode == "f32" else L.PV_F16
    if Nq == Nk and layout == "slices":
        buf = torch.cat([q, k, v], -1).to(tdt).to(_dev()).contiguous()
        qp, kp, vp = (buf.data_ptr() + i * D * buf.element_size() for i in range(3))
        q_rs = kv_rs = 3 * D
        q_bs = kv_bs = Nq * 3 * D
    else:
        qb = q.to(tdt).to(_dev()).contiguous()
        buf = torch.cat([k, v], -1).to(tdt).to(_dev()).contiguous()
        qp, kp, vp = qb.data_ptr(), buf.data_ptr(), buf.data_ptr() + D * buf.element_size()
        q_rs, kv_rs, q_bs, kv_bs = D, 2 * D, Nq * D, Nk * 2 * D
    off = 1 if mode == "unaligned" else 0
    o = torch.empty(off + B * Nq * D, dtype=tdt, device=_dev())
    d = _desc(dt, B, Nq, Nk, D, q_rs, kv_rs, q_bs, kv_bs, D, Nq * D, normalize, 1 if resid else 0, scale)
    L.check(L.load().pv_attention_fwd(C.byref(d), qp, kp, vp, o.data_ptr() + off * o.element_size(),
                                      torch.cuda.current_stream().cuda_stream), "pv_attention_fwd")
    torch.cuda.synchronize()
    return o[off:].view(B, Nq, D).float().cpu()


def _qkv(B, Nq, Nk, D, seed, mag=1.0):
    g = torch.Generator().manual_seed(seed)
    return tuple(TS.f16_exact(torch.randn(B, n, D, generator=g) * mag) for n in (Nq, Nk, Nk))


@pytest.mark.gpu
@pytest.mark.parametrize("row", WIDE_ROWS, ids=["%s-%s-m%d-%dx%d-b%d" % (r[0], r[1], r[3], r[4], r[5], r[6]) for r in WIDE_ROWS])
def test_wide_attention_instance(row):
    name, mode, D, normalize, Nq, Nk, B = row
    q, k, v = _qkv(B, Nq, Nk, D, seed=D + 7 * Nq + Nk + normalize)
    scale = D ** -0.5 if not normalize else 1.0
    ref, absref = _ref64(q, k, v, scale, normalize)
    got, launched = TS.launched_kernels(_run_attention, q, k, v, scale, normalize, mode)
    assert name in launched, "expected %s, launched %s" % (name, launched)
    if mode != "f32":
        ratio = TS.assert_close_to_f64(got, ref, absref, 0, acc_eps=ACC_EPS_ATTN, what=name)
    else:
        # fp32 storage and maths: only fp32 summation and __expf rounding remain
        err = (got.double() - ref).abs()
        tol = 1e-5 * absref + 1e-30
        ratio = (float((err / tol).max()), 0.0)
        assert ratio[0] <= 1.0, float(err.max())
    print("RATIO attention-wide %s-%s-m%d-%dx%d %.4f %.4f" % (name, mode, normalize, Nq, Nk, ratio[0], ratio[1]))


@pytest.mark.gpu
@pytest.mark.parametrize("D,mode", [(256, "f16"), (512, "f16"), (256, "f32"), (512, "f32")])
def test_wide_softmax_late_maximum(D, mode):
    """As the kernel matrix's attention-late-max: every query's largest key sits in the last (partial) key tile and
    all earlier tiles score ~100 below it, so the running-max correction factor underflows to 0 when it arrives."""
    B, Nq, Nk = 1, 70, 200
    g = torch.Generator().manual_seed(D)
    scale = D ** -0.5
    u = torch.randn(1, 1, D, generator=g)
    q = TS.f16_exact(2 * u + 0.5 * torch.randn(B, Nq, D, generator=g))
    k = TS.f16_exact(torch.randn(B, Nk, D, generator=g) * 0.05)
    v = TS.f16_exact(torch.randn(B, Nk, D, generator=g))
    c = 50.0 / (scale * 2 * float((u * u).sum()))
    k[:, 197] = TS.f16_exact(c * u[0, 0])
    k[:, :192] = TS.f16_exact(-c * u[0, 0])
    logits = (q.double() @ k.double().transpose(-2, -1)) * scale
    assert bool((logits.argmax(-1) == 197).all())
    assert float((logits[..., :192].max(-1).values - logits[..., 197]).max()) < -88
    ref, absref = _ref64(q, k, v, scale, 0, resid=True)
    got, launched = TS.launched_kernels(_run_attention, q, k, v, scale, 0, mode, "dense", True)
    name = ("attention_wide_kernel<%d,256>" % D) if mode == "f16" else "attention_wide_simt_kernel<float,%d>" % D
    assert name in launched, launched
    if mode == "f16":
        TS.assert_close_to_f64(got, ref, absref, 0, acc_eps=ACC_EPS_ATTN, what=name)
    else:
        assert bool(((got.double() - ref).abs() <= 1e-5 * absref + 1e-6).all())


@pytest.mark.gpu
@pytest.mark.parametrize("D", [64, 128, 256, 512])
def test_wide_linear_large_magnitude(D):
    """Linear mode with |q.k| in the thousands: the division by Nk happens in fp32 before P is rounded to f16, so
    neither S nor P overflows f16 and the result stays inside the f64 bound."""
    B, Nq, Nk = 2, 130, 63
    q, k, _ = _qkv(B, Nq, Nk, D, seed=5 * D, mag=48.0)
    v = TS.f16_exact(torch.randn(B, Nk, D, generator=torch.Generator().manual_seed(D)) * 0.05)
    s = q.double() @ k.double().transpose(-2, -1)
    assert float(s.abs().max()) > 60000                      # S itself would not fit in f16
    ref, absref = _ref64(q, k, v, 1.0, 1)
    assert float(ref.abs().max()) < 60000
    got, launched = TS.launched_kernels(_run_attention, q, k, v, 1.0, 1, "f16")
    dout = min(D, 256)
    assert "attention_wide_kernel<%d,%d>" % (D, dout) in launched, launched
    TS.assert_close_to_f64(got, ref, absref, 0, acc_eps=ACC_EPS_ATTN, what="linear-large-D%d" % D)


@pytest.mark.gpu
@pytest.mark.parametrize("D,normalize,mode", [(64, 1, "f16"), (128, 1, "f16"), (256, 0, "f16"), (256, 1, "f16"),
                                              (512, 0, "f16"), (512, 1, "f16"), (512, 0, "f32"), (256, 1, "unaligned")])
def test_wide_batch_invariance(D, normalize, mode):
    """B = 3 gives bit for bit the three B = 1 results."""
    q, k, v = _qkv(3, 196, 784, D, seed=D + normalize)
    scale = 1.0 if normalize else D ** -0.5
    full = _run_attention(q, k, v, scale, normalize, mode)
    for b in range(3):
        one = _run_attention(q[b:b + 1], k[b:b + 1], v[b:b + 1], scale, normalize, mode)
        assert torch.equal(full[b:b + 1], one), (b, float((full[b:b + 1] - one).abs().max()))


# ---- GPU layer cases -------------------------------------------------------------------------------------------------
def _expected_core(case):
    kw, _ = TS.NONLOCAL_CASES[case]
    di, lin = kw["dim_inner"], kw.get("instantiation", "softmax") == "dot_product"
    if di >= 256:
        return "attention_wide_kernel<%d,256>" % di
    if lin:
        return "attention_wide_kernel<%d,%d>" % (di, di)
    return "attention_mma_kernel<128>" if di == 128 else "attention_wgmma_kernel<%d>" % di


def _expected_core_f32(case):
    kw, _ = TS.NONLOCAL_CASES[case]
    di, lin = kw["dim_inner"], kw.get("instantiation", "softmax") == "dot_product"
    return ("attention_wide_simt_kernel<float,%d>" if (di >= 256 or lin) else "attention_kernel<float,%d>") % di


def _build(case):
    from pytorchvideo_b200.layers.nonlocal_net import create_nonlocal
    m, x = TS.build_nonlocal_case(case, create_nonlocal, seed=GOLD[case]["seed"])
    assert abs(TS.state_checksum(m) - GOLD[case]["state_checksum"]) <= 1e-6 * abs(GOLD[case]["state_checksum"])
    return m, x


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(TS.NONLOCAL_CASES))
def test_nonlocal_layer_f16(case):
    m, x = _build(case)
    ref = GOLD[case]["output"]
    m = m.cuda()
    out, launched = TS.launched_kernels(lambda: m(x.cuda()).float().cpu())
    assert _expected_core(case) in launched, launched
    assert out.shape == ref.shape
    scale = float(ref.abs().max())
    err = (out - ref).abs()
    inside = float((err <= 1e-3 * ref.abs() + 1e-4 * max(1.0, scale)).float().mean())
    print("PARITY nonlocal %s f16: max|d|/max|ref| = %.3e, in-band %.3f" % (case, float(err.max()) / scale, inside))
    assert bool((err <= 2e-3 * ref.abs() + 1e-3 * scale).all()), float(err.max()) / scale


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(TS.NONLOCAL_CASES))
def test_nonlocal_layer_f32_parity_mode(case):
    from pytorchvideo_b200 import config
    m, x = _build(case)
    ref = GOLD[case]["output"]
    config.set_precision("f32")
    try:
        m = m.cuda()
        out, launched = TS.launched_kernels(lambda: m(x.cuda()).float().cpu())
    finally:
        config.set_precision("f16")
    assert _expected_core_f32(case) in launched, launched
    scale = max(1.0, float(ref.abs().max()))
    assert bool(((out - ref).abs() <= 1e-3 * ref.abs() + 1e-4 * scale).all()), float((out - ref).abs().max())


@pytest.mark.gpu
def test_nonlocal_transmute_route():
    from pytorchvideo_b200.accelerator import transmute_model
    from pytorchvideo_b200.accelerator.b200 import B200Block
    case = "softmax_pool_512_256"
    m, x = _build(case)
    wrap = nn.Sequential(m)
    transmute_model(wrap, "b200")
    assert isinstance(wrap[0], B200Block)
    out = wrap.cuda()(x.cuda()).float().cpu()
    ref = GOLD[case]["output"]
    scale = float(ref.abs().max())
    assert bool(((out - ref).abs() <= 2e-3 * ref.abs() + 1e-3 * scale).all())


# ---- GPU model: i3d_r50 with the I3D-NLN layout of Non-local blocks ----------------------------------------------
def _i3d_nln():
    import pytorchvideo_b200.models.hub as PH
    from pytorchvideo_b200.layers.nonlocal_net import create_nonlocal
    return TS.build_i3d_nln(PH, create_nonlocal)


# (min fraction of logits inside rtol 1e-3 / atol 1e-4*scale, max |d|/max|ref|): measured values with a small margin.
# First H100 run (NVIDIA H100 80GB HBM3, 700 W power limit): in-band 0.3425, max |d|/max|ref| 2.949e-3.
I3D_NLN_F16_BOUNDS = (0.32, 3.3e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["f32", "f16"])
def test_i3d_r50_with_nonlocal_blocks(precision):
    from pytorchvideo_b200 import config
    model, clip = _i3d_nln()
    ref = nonlocal_forward(model, clip)
    config.set_precision(precision)
    try:
        model.cuda()
        out, launched = TS.launched_kernels(lambda: model(clip.cuda()).float().cpu())
    finally:
        config.set_precision("f16")
        model.cpu()
    if precision == "f16":
        assert "attention_wide_kernel<256,256>" in launched and "attention_wide_kernel<512,256>" in launched, launched
    else:
        assert "attention_wide_simt_kernel<float,256>" in launched and "attention_wide_simt_kernel<float,512>" in launched
    scale = max(1.0, float(ref.abs().max()))
    err = (out - ref).abs()
    tol = 1e-3 * ref.abs() + 1e-4 * scale
    inside = float((err <= tol).float().mean())
    print("PARITY i3d_r50+NL %s: max|d|/max|ref| = %.3e, in-band %.4f" % (precision, float(err.max()) / scale, inside))
    assert out.shape == ref.shape
    if precision == "f32":
        assert bool((err <= tol).all()), "max err %.3e (scale %.3g)" % (float(err.max()), scale)
    else:
        assert inside >= I3D_NLN_F16_BOUNDS[0] and float(err.max()) / scale <= I3D_NLN_F16_BOUNDS[1]
