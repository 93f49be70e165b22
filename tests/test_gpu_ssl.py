"""GPU: the self-supervised objectives (csrc/pv_contrastive.cu) and the SimCLR / BYOL / MemoryBank /
SoftTargetCrossEntropyLoss wrappers on an H100.

Every test asserts which kernel instances ran (pv_kernel_counts).
- Bit-exact: pv_ema_update against the reference's eager expression and BYOL's momentum parameters against the
  reference's after a call; MemoryBank's drawn indices; repeated calls.
- Bounded against float64, with the bound derived next to each test: pv_rows_l2_normalize, pv_contrastive_ce (SimCLR
  and BYOL modes, a gathered key block with a target offset), pv_memory_bank_ce (K not a multiple of the warp, dims
  2 .. 2048, an out-of-range index, a bank above 2^31 elements), pv_soft_target_ce.
- End to end against tests/golden/ssl.pt (the reference on the CPU).  f32 precision: losses within 2e-4 relative (+1e-5
  absolute) and embeddings within 2e-4.  f16 precision (the trunk and projector in f16 storage, the objectives in
  fp32): losses within 3e-2 relative (+2e-3 absolute) and embeddings within 3e-2 absolute.  Largest err / tol
  measured on an H100 80GB HBM3: f32 0.003 (losses and embeddings); f16 0.18 (loss) and 0.21 (embedding), both in
  memory_bank_unit, whose 2-wide embedding at T = 0.07 is the most sensitive case.
"""
import copy
import hashlib
import math
import os
import types

import pytest
import torch
import torch.nn as nn

from pytorchvideo_b200 import config, contrastive as K, testing as TS
from pytorchvideo_b200.layers import make_multilayer_perceptron
from pytorchvideo_b200.losses import SoftTargetCrossEntropyLoss
from pytorchvideo_b200.models.byol import BYOL
from pytorchvideo_b200.models.memory_bank import MemoryBank
from pytorchvideo_b200.models.resnet import create_resnet
from pytorchvideo_b200.models.simclr import SimCLR

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ssl.pt")
NS = types.SimpleNamespace(SimCLR=SimCLR, BYOL=BYOL, MemoryBank=MemoryBank, create_resnet=create_resnet,
                           make_multilayer_perceptron=make_multilayer_perceptron)
EPS = 2.0 ** -24
DEV = "cuda"


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)


def _ran(counts, *names):
    for n in names:
        assert counts.get(n, 0) >= 1, "%s did not run: %s" % (n, counts)


def _unit_rows(n, c, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((n, c), generator=g, dtype=torch.float64)
    return x / x.norm(dim=1, keepdim=True)


# ---- pv_ema_update: bit-exact against p_m * mmt + p * (1.0 - mmt) in eager fp32 -------------------------------------
def test_ema_update_bit_exact():
    g = torch.Generator().manual_seed(3)
    shapes = [(7,), (4096,), (4097,), (3, 5, 7, 11), (64, 2048)]
    src = [torch.randn(s, generator=g) for s in shapes]
    dst = [torch.randn(s, generator=g) for s in shapes]
    for mmt in (0.99, 0.996, 0.5):
        want = [d * mmt + s * (1.0 - mmt) for d, s in zip(dst, src)]
        dd = [d.to(DEV) for d in dst]
        upd = K.EmaUpdate(dd, [s.to(DEV) for s in src])
        _, counts = TS.launched_kernels(upd, mmt)
        _ran(counts, "ema_update_kernel")
        for a, b in zip(dd, want):
            assert torch.equal(a.cpu(), b)


# ---- pv_rows_l2_normalize: sum of C squares in fp32 (relative error <= C u), sqrt (+u, halves the sum's error), one
#      division (+u): |y - y64| <= (C / 2 + 2) u |y64| + 1e-38 ----------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("rows,C", [(3, 2), (257, 4), (5, 128), (33, 2048)])
def test_l2_normalize_vs_f64(dtype, rows, C):
    g = torch.Generator().manual_seed(rows * C)
    x = (torch.randn((rows, C), generator=g) * 3).to(dtype)
    x[0] = 0                                                        # the 1e-12 clamp: zeros stay zeros
    ref = x.double() / x.double().norm(dim=1, keepdim=True).clamp_min(1e-12)
    y, counts = TS.launched_kernels(K.l2_normalize, x.to(DEV))
    _ran(counts, "l2_normalize_kernel<%s>" % ("float" if dtype == torch.float32 else "__half"))
    err = (y.cpu().double() - ref).abs()
    tol = (C / 2 + 2) * EPS * ref.abs() + 1e-38
    print("RATIO l2_normalize %s %dx%d %.3f" % (dtype, rows, C, float((err / tol).max())))
    assert bool((err <= tol).all())


# ---- pv_contrastive_ce.  Unit rows: |q . k| <= 1 with an fp32 error <= (C + 1) u; divided by T (+u): each logit within
#      d = ((C + 2) u) / T.  logsumexp moves by at most max d, plus the fp32 sum of M exponentials (M u relative -> M u
#      absolute in the log), expf / logf (4 u), the final subtraction (u |row|); the mean of N rows adds N u |loss|.
def _ce_tol(C, M, N, T, loss):
    return 2 * (2 * (C + 2) * EPS / T + (M + 8) * EPS + (N + 4) * EPS * abs(loss) + 4 * EPS * (1 / T))


@pytest.mark.parametrize("N,M,off,C", [(3, 3, 0, 2), (1, 1, 0, 4), (32, 64, 32, 128), (37, 111, 74, 2048),
                                       (8, 4096, 4000, 128)])
def test_simclr_ce_vs_f64(N, M, off, C):
    T = 0.07
    q, k = _unit_rows(N, C, 1), _unit_rows(M, C, 2)
    k[off:off + N] = 0.6 * q + 0.8 * _unit_rows(N, C, 3)              # positives that score above the negatives
    k = k / k.norm(dim=1, keepdim=True)
    logits = q @ k.T / T
    ref = float((torch.logsumexp(logits, 1) - logits[torch.arange(N), off + torch.arange(N)]).mean())
    got, counts = TS.launched_kernels(K.contrastive_ce, q.float().to(DEV), k.float().to(DEV), T, off)
    _ran(counts, "contrastive_rows_kernel<simclr>", "mean_kernel")
    tol = _ce_tol(C, M, N, T, ref)
    print("RATIO simclr_ce N=%d M=%d C=%d %.3f" % (N, M, C, abs(float(got) - ref) / tol))
    assert abs(float(got) - ref) <= tol


@pytest.mark.parametrize("N,C", [(2, 4), (33, 128), (64, 2048)])
def test_byol_ce_vs_f64(N, C):
    q, k = _unit_rows(N, C, 4), _unit_rows(N, C, 5)
    ref = float(-(q * k).sum(1).mean())
    got, counts = TS.launched_kernels(K.contrastive_ce, q.float().to(DEV), k.float().to(DEV), 1.0, 0, True)
    _ran(counts, "contrastive_rows_kernel<byol>", "mean_kernel")
    tol = 2 * ((C + 2) * EPS + (N + 2) * EPS)
    assert abs(float(got) - ref) <= tol


def test_contrastive_ce_refuses_bad_target():
    q = torch.zeros(4, 8, device=DEV)
    with pytest.raises(RuntimeError):
        K.contrastive_ce(q, q, 0.07, 1)                  # targets 1 .. 4 of 4 keys


# ---- pv_memory_bank_ce: logits as in pv_contrastive_ce (bank rows are not unit rows: |m . x| <= |m| |x|), K1 = K rows
def _mb_ref(x, mem, idx, T):
    w = mem[idx]                                          # (B, K1, dim) float64
    logits = torch.einsum("bkc,bc->bk", w, x) / T
    mag = torch.einsum("bkc,bc->bk", w.abs(), x.abs()) / T
    return float((torch.logsumexp(logits, 1) - logits[:, 0]).mean()), float(mag.max())


@pytest.mark.parametrize("B,K1,dim", [(3, 37, 2), (2, 4097, 4), (4, 65, 128), (3, 1000, 2048), (5, 33, 130)])
def test_memory_bank_ce_vs_f64(B, K1, dim):
    T = 0.07
    g = torch.Generator().manual_seed(K1 + dim)
    bank = 5000
    mem = (torch.rand((bank, dim), generator=g) * 2 - 1) / math.sqrt(dim / 3)
    x = _unit_rows(B, dim, 6)
    idx = torch.randint(0, bank, (B, K1), generator=g)
    ref, mag = _mb_ref(x, mem.double(), idx, T)
    got, counts = TS.launched_kernels(K.memory_bank_ce, x.float().to(DEV), mem.to(DEV), idx.to(DEV), T)
    vec = "vec4" if dim % 4 == 0 else "scalar"
    _ran(counts, "memory_bank_logits_kernel<%s>" % vec, "lse_target0_kernel", "mean_kernel")
    tol = 2 * (2 * (dim + 2) * EPS * mag + (K1 + 8) * EPS + (B + 4) * EPS * abs(ref) + 4 * EPS / T)
    print("RATIO memory_bank_ce B=%d K1=%d dim=%d %.3f" % (B, K1, dim, abs(float(got) - ref) / tol))
    assert abs(float(got) - ref) <= tol
    again = K.memory_bank_ce(x.float().to(DEV), mem.to(DEV), idx.to(DEV), T)
    assert torch.equal(got, again)


def test_memory_bank_ce_out_of_range_raises():
    mem = torch.rand((16, 8), device=DEV)
    x = torch.rand((2, 8), device=DEV)
    for bad in (16, -1, 1 << 40):
        idx = torch.zeros((2, 5), dtype=torch.int64)
        idx[1, 3] = bad
        with pytest.raises(RuntimeError, match="out of range"):
            K.memory_bank_ce(x, mem, idx.to(DEV), 0.07)


def test_memory_bank_ce_64bit_offsets():
    dim = 2048
    rows = (1 << 31) // dim + 64                          # > 2^31 elements: byte offsets need 64 bits
    need = rows * dim * 4 + (1 << 28)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip("needs %.1f GB of free device memory" % (need / 1e9))
    mem = torch.empty((rows, dim), dtype=torch.float32, device=DEV)
    g = torch.Generator().manual_seed(11)
    tail = torch.rand((8, dim), generator=g) - 0.5
    head = torch.rand((8, dim), generator=g) - 0.5
    mem[-8:] = tail.to(DEV)
    mem[:8] = head.to(DEV)
    x = _unit_rows(2, dim, 7)
    idx = torch.tensor([[rows - 1, rows - 8, 3, rows - 2], [rows - 3, 0, rows - 5, 7]])
    small = torch.cat([head, tail]).double()
    remap = torch.where(idx >= rows - 8, idx - (rows - 8) + 8, idx)
    ref, mag = _mb_ref(x, small, remap, 0.07)
    got, counts = TS.launched_kernels(K.memory_bank_ce, x.float().to(DEV), mem, idx.to(DEV), 0.07)
    _ran(counts, "memory_bank_logits_kernel<vec4>")
    assert abs(float(got) - ref) <= 2 * (2 * (dim + 2) * EPS * mag + 16 * EPS + 8 * EPS * abs(ref) + 60 * EPS)
    del mem
    torch.cuda.empty_cache()


# ---- pv_soft_target_ce against the reference's values and float64.  Per row, in the kernel's order (u = 2^-24):
#      m = max x exactly; se = sum_c expf(x_c - m): C fp32 additions and expf's 2 ulp, so lz = logf(se) is off by at most
#      (C + 4) u (relative error of se, carried into the log) + u |lz| (logf);  ls_c = (x_c - m) - lz: two roundings,
#      u |x_c - m| + u |ls_c|, plus the error of lz;  t_c / (eps + sum t): the sum of C targets and the division, a
#      relative (C + 2) u;  acc = sum_c fmaf(-t_c, ls_c, acc): C roundings, C u sum |t_c ls_c|.  Together
#        tol_row = (2 C + 4) u sum_c |t_c ls_c| + sum_c |t_c| ((C + 4) u + u |lz| + u |x_c - m|)
#      with t the (normalised) targets; the mean adds (N + 2) u |mean| and carries the average of the row bounds.
#      A factor 2 covers the float64 reference's own rounding and leaves margin.
@pytest.mark.parametrize("name", list(TS.SOFT_CE_CASES))
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_soft_target_ce(gold, name, dtype):
    x, t, kw = TS.soft_ce_case(name)
    x = x.to(dtype)
    loss = SoftTargetCrossEntropyLoss(**kw)
    got, counts = TS.launched_kernels(loss, x.to(DEV), t.to(DEV))
    xt = "float" if dtype == torch.float32 else "__half"
    _ran(counts, "soft_target_rows_kernel<%s,%s>" % (xt, "int64" if t.dim() == 1 else "float"))
    x64 = x.double()
    N, C = x.shape
    t64 = torch.nn.functional.one_hot(t, C).double() if t.dim() == 1 else t.double()
    if kw["normalize_targets"]:
        t64 = t64 / (torch.finfo(torch.float32).eps + t64.sum(1, keepdim=True))
    ls = torch.log_softmax(x64, 1)
    per = -(t64 * ls).sum(1)
    xm = x64 - x64.max(1, keepdim=True).values
    lz = torch.logsumexp(xm, 1, keepdim=True)
    row_tol = ((2 * C + 4) * EPS * (t64 * ls).abs().sum(1)
               + (t64.abs() * ((C + 4) * EPS + EPS * lz.abs() + EPS * xm.abs())).sum(1))
    if kw["reduction"] == "mean":
        ref = per.mean()
        tol = 2 * (row_tol.mean() + (N + 2) * EPS * ref.abs())
    else:
        ref, tol = per, 2 * row_tol
    err = (got.cpu().double() - ref).abs()
    tol = tol + 1e-30
    ratio = float((err / tol).max())
    print("RATIO soft_ce %s %s %.3f (tol/|loss| %.1e)" % (name, dtype, ratio, float((tol / ref.abs().clamp_min(1e-30)).max())))
    assert ratio <= 1
    if dtype == torch.float32:                # the reference's own fp32 result: both within their bounds of float64
        assert bool(((got.cpu().double() - gold["soft_ce"][name].double()).abs() <= 2 * tol).all())
    assert got.shape == ((N,) if kw["reduction"] == "none" else ())


# ---- end to end against the reference --------------------------------------------------------------------------------
def _run_case(name, gold, precision):
    config.set_precision(precision)
    try:
        m, args = TS.build_ssl_case(name, NS)
        m = m.to(DEV)
        args = tuple(a.to(DEV) for a in args)
        out = {}
        if name.startswith("byol"):
            out["embedding"] = m.forward_backbone(args[0])
        else:
            out["embedding"] = m.embed(args[0])
        torch.manual_seed(77)
        loss, counts = TS.launched_kernels(m, *args)
        out["loss"] = float(loss)
        out["counts"] = counts
        out["model"] = m
        out["args"] = args
        assert loss.dim() == 0 and loss.dtype == torch.float32 and loss.device.type == "cuda"
        return out
    finally:
        config.set_precision("f16")


CASE_KERNELS = {"simclr": ("l2_normalize_kernel<float>", "contrastive_rows_kernel<simclr>"),
                "byol": ("ema_update_kernel", "l2_normalize_kernel<float>", "contrastive_rows_kernel<byol>",
                         "refresh_gather_kernel", "refresh_fold_kernel"),
                "memory_bank": ("l2_normalize_kernel<float>", "lse_target0_kernel")}


@pytest.mark.parametrize("precision", ["f32", "f16"])
@pytest.mark.parametrize("name", TS.SSL_CASES)
def test_end_to_end_vs_reference(gold, name, precision):
    g = gold["cases"][name]
    out = _run_case(name, gold, precision)
    config.set_precision(precision)
    try:
        _check_case(g, name, precision, out)
    finally:
        config.set_precision("f16")


def _check_case(g, name, precision, out):
    _ran(out["counts"], *CASE_KERNELS["memory_bank" if name.startswith("memory") else name.split("_")[0]])
    rl, al, ae = (2e-4, 1e-5, 2e-4) if precision == "f32" else (3e-2, 2e-3, 3e-2)
    lerr = abs(out["loss"] - g["loss"])
    eerr = float((out["embedding"].cpu() - g["embedding"]).abs().max())
    print("RATIO e2e %s %s loss_err=%.3e (%.3f) emb_err=%.3e (%.3f)" % (
        name, precision, lerr, lerr / (rl * abs(g["loss"]) + al), eerr, eerr / ae))
    assert lerr <= rl * abs(g["loss"]) + al
    assert eerr <= ae
    if name.startswith("byol"):
        m = out["model"]
        got = [hashlib.sha256(p.detach().cpu().numpy().tobytes()).hexdigest() for p in m.backbone_mmt.parameters()]
        if g["mmt_param_values"] is not None:
            for p, want in zip(m.backbone_mmt.parameters(), g["mmt_param_values"]):
                assert torch.equal(p.detach().cpu(), want)       # the EMA is bit-exact to the reference's
        else:
            assert got == g["mmt_params"]                    # bit-exact, as sha256 of the bytes
        # the momentum plan after the update (refreshed in place) against the reference's momentum backbone
        emb = m.forward_backbone_mmt(out["args"][0])
        merr = float((emb.cpu() - g["embedding_mmt_after"]).abs().max())
        print("RATIO e2e %s %s mmt_emb_err=%.3e (%.3f)" % (name, precision, merr, merr / ae))
        assert merr <= ae
    if name.startswith("memory_bank"):
        m, (x, x_ind) = out["model"], out["args"]
        torch.manual_seed(77)
        assert torch.equal(m.draw_indices(x.shape[0], x_ind, DEV).cpu(), g["indices"])


@pytest.mark.parametrize("name", ["simclr_video", "memory_bank_unit", "simclr_unit"])
def test_repeated_calls_bitwise_identical(name):
    m, args = TS.build_ssl_case(name, NS)
    m = m.to(DEV)
    args = tuple(a.to(DEV) for a in args)
    vals = []
    for _ in range(3):
        torch.manual_seed(77)
        vals.append(m(*args).cpu())
    assert all(torch.equal(vals[0], v) for v in vals[1:])


@pytest.mark.parametrize("precision", ["f32", "f16"])
@pytest.mark.parametrize("name", ["byol_unit_mmt", "byol_video"])
def test_byol_momentum_plan_refreshed_in_place(name, precision, monkeypatch):
    """The momentum plan is compiled once and refreshed in place (pv_weights_refresh): after every call its output
    equals, bit for bit, that of a freshly compiled plan of the updated momentum backbone, and the same plan and CUDA
    graph object are replayed with no compile.  The online backbone is given weights of its own and mmt = 0.5, so every
    update moves the momentum weights far."""
    from pytorchvideo_b200.engine import lower as LW
    config.set_precision(precision)
    try:
        m, (x1, x2) = TS.build_ssl_case(name, NS)
        if name == "byol_video":
            TS.randomize_model(m.backbone, seed=99)
            m.update_mmt(0.5)
        m = m.to(DEV)
        x1, x2 = x1.to(DEV), x2.to(DEV)
        compiles = []
        real = LW.compile_model
        monkeypatch.setattr(LW, "compile_model", lambda *a, **k: compiles.append(1) or real(*a, **k))
        plan = graph = None
        for step in range(3):
            n0 = len(compiles)
            _, counts = TS.launched_kernels(m, x1, x2)
            assert len(compiles) - n0 == (1 if step == 0 else 0)        # compiled on the first call only
            (cm, refresh), = m._state()["plans"].values()
            assert refresh is not None, "the momentum plan is not refreshable"
            _ran(counts, "ema_update_kernel", "refresh_gather_kernel", "refresh_fold_kernel")
            if step == 0:
                plan, graph = cm, cm.graph
            else:
                assert cm is plan and cm.graph is graph and graph is not None
            got = m.forward_backbone_mmt(x1)
            fresh = copy.deepcopy(m)                       # compiles its own momentum plan
            want = fresh.forward_backbone_mmt(x1)
            assert torch.equal(got, want), step
            del fresh
    finally:
        config.set_precision("f16")
