"""GPU: the bank scans of csrc/pv_bank.cu (KnnMemory.eval_knn / update and MoCo's queue cross entropy) on an H100.

Every test asserts which kernel instances ran (pv_kernel_counts).
- Bit-exact: pv_bank_update against the reference's eager expression on the CPU (|v| < 1e-12, +-0, NaN, +-inf,
  repeated indices), repeated calls.
- kNN against float64: a similarity sums dim fp32 products with fmaf, so |s - s64| <= tol = (dim + 2) u sum_c |q_c m_c|
  (u = 2^-24).  The returned set must be a valid top-k within that band: descending, each returned similarity within
  tol of its float64 value, and no bank row left out whose float64 similarity exceeds the smallest returned one by more
  than 2 tol.  Equal similarities must come out by ascending index.  The vote is compared with float64 over the
  returned set: each weight exp(s / T) carries the division and expf (3 u relative), the k-term sum k u.
- Queue cross entropy against float64: logits within ((dim + 2) u mag + u) / T, the logsumexp adds the K-term sum and
  the slab combination, see _ce_tol.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from pytorchvideo_b200 import contrastive as K, testing as TS
from pytorchvideo_b200.losses import ContrastiveLoss
from pytorchvideo_b200.models.knn_memory import KnnMemory

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -24
DEV = "cuda"


def _ran(counts, *names):
    for n in names:
        assert counts.get(n, 0) >= 1, "%s did not run: %s" % (n, counts)


def _unit_rows(n, c, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((n, c), generator=g)
    return x / x.norm(dim=1, keepdim=True)


def _score_name(k, dim):
    return "bank_score_kernel<topk,%d,%s>" % (32 if k <= 256 else 8, "vec4" if dim % 4 == 0 else "scalar")


# ---- pv_bank_update: bit-exact against the reference's expression ----------------------------------------------------
def _update_ref(memory, mem, ind, momentum):
    """ssl_helper.py:245-250 on the CPU, on one thread: there index_put_ keeps the last occurrence of a repeated index.
    With several threads torch splits the indices into chunks that run concurrently, and a repeated index whose
    occurrences fall in different chunks can keep an earlier one."""
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        memory = memory.clone()
        mem = mem.view(mem.size(0), 1, -1)
        old = memory[ind.view(-1), :].view(ind.size(0), -1, memory.shape[1])
        upd = F.normalize(mem * momentum + old * (1 - momentum), p=2, dim=1)
        memory[ind.view(-1), :] = upd.squeeze()
        return memory
    finally:
        torch.set_num_threads(threads)


@pytest.mark.parametrize("momentum", [1.0, 0.5, 0.996])
@pytest.mark.parametrize("N,M,dim", [(1, 10, 128), (64, 1000, 128), (300, 50, 7), (5, 5, 2048)])
def test_bank_update_bit_exact(momentum, N, M, dim):
    g = torch.Generator().manual_seed(N * M + dim)
    memory = torch.rand((M, dim), generator=g) * 2 - 1
    mem = torch.randn((N, dim), generator=g)
    mem[0, :4] = torch.tensor([0.0, -0.0, 1e-13, -3e-30])
    memory[:, 4:6] = torch.tensor([float("nan"), 1e-20])
    if dim > 8:
        mem[-1, 8] = float("inf")
    ind = torch.randint(0, M, (N,), generator=g)
    ind[-1] = ind[0]                                       # a repeated index: the last occurrence wins
    want = _update_ref(memory, mem, ind, momentum)
    got = memory.to(DEV)
    _, counts = TS.launched_kernels(K.bank_update, got, mem.to(DEV), ind.to(DEV), momentum)
    _ran(counts, "bank_update_kernel")
    _assert_same_bits(got.cpu(), want)


def _assert_same_bits(a, b):
    """Bit for bit, except that a NaN may carry any payload (x86 and the GPU make different default NaNs)."""
    na, nb = torch.isnan(a), torch.isnan(b)
    assert torch.equal(na, nb)
    assert torch.equal(a[~na].view(torch.int32), b[~nb].view(torch.int32))


def test_bank_update_many_duplicates_last_wins():
    g = torch.Generator().manual_seed(5)
    memory = torch.rand((10, 16), generator=g)
    mem = torch.randn((5000, 16), generator=g)
    ind = torch.randint(0, 10, (5000,), generator=g)
    want = _update_ref(memory, mem, ind, 0.5)
    got = memory.to(DEV)
    _, counts = TS.launched_kernels(K.bank_update, got, mem.to(DEV), ind.to(DEV), 0.5)
    _ran(counts, "bank_update_kernel")
    _assert_same_bits(got.cpu(), want)


def test_bank_update_out_of_range_writes_nothing():
    memory = torch.rand((16, 8), device=DEV)
    before = memory.clone()
    for bad in (16, -1):
        ind = torch.tensor([3, bad, 5], device=DEV)
        with pytest.raises(RuntimeError, match="out of range"):
            K.bank_update(memory, torch.rand((3, 8), device=DEV), ind, 0.5)
        assert torch.equal(memory, before)


# ---- pv_bank_topk against float64 ------------------------------------------------------------------------------------
def _check_topk(q, mem, labels, k, C, T, sims, idx, preds):
    q64, m64 = q.double(), mem.double()
    s64 = q64 @ m64.T
    tol = (q.shape[1] + 2) * EPS * (q64.abs() @ m64.abs().T) + 1e-30
    sims, idx, preds = sims.cpu().double(), idx.cpu(), preds.cpu().double()
    N = q.shape[0]
    ratio = 0.0
    for n in range(N):
        assert len(set(idx[n].tolist())) == k
        assert bool((sims[n][1:] <= sims[n][:-1]).all()), "not descending"
        got64 = s64[n][idx[n]]
        t = tol[n][idx[n]]
        ratio = max(ratio, float(((sims[n] - got64).abs() / t).max()))
        assert bool(((sims[n] - got64).abs() <= t).all())
        out = torch.ones(mem.shape[0], dtype=torch.bool)
        out[idx[n]] = False
        if out.any():
            floor = float(got64.min())
            worst = float((s64[n][out] - tol[n][out]).max()) - float(t.max())
            assert worst <= floor, "row %d: a left-out row scores %.9g above the k-th %.9g" % (n, worst, floor)
        eq = sims[n][1:] == sims[n][:-1]                   # ties: ascending bank index
        assert bool((idx[n][1:][eq] > idx[n][:-1][eq]).all())
        # each weight: the fp32 T and the division move the exponent by 2 u |s / T|, expf adds 2 u; the sum k u
        w = torch.exp(sims[n] / T)
        wt = w * ((k + 4) * EPS + 2 * EPS * (sims[n] / T).abs())
        want = torch.zeros(C, dtype=torch.float64).index_add_(0, labels[idx[n]], w)
        ptol = 2 * torch.zeros(C, dtype=torch.float64).index_add_(0, labels[idx[n]], wt) + 1e-38
        assert bool(((preds[n] - want).abs() <= ptol).all()), float(((preds[n] - want).abs() / ptol).max())
    return ratio


@pytest.mark.parametrize("N,M,dim,k,kernel", [
    (3, 1000, 8, 1, "bank_score_kernel<topk,32,vec4>"), (5, 1000, 100, 20, "bank_score_kernel<topk,32,vec4>"),
    (4, 1000, 128, 1000, "bank_score_kernel<topk,8,vec4>"), (2, 1000, 128, 256, "bank_score_kernel<topk,32,vec4>"),
    (33, 4099, 64, 7, "bank_score_kernel<topk,32,vec4>"), (2, 5000, 130, 1024, "bank_score_kernel<topk,8,scalar>"),
    (9, 777, 3, 300, "bank_score_kernel<topk,8,scalar>"), (1, 1, 5, 1, "bank_score_kernel<topk,32,scalar>"),
    (6, 3000, 50, 40, "bank_score_kernel<topk,32,scalar>")])
def test_bank_topk_vs_f64(N, M, dim, k, kernel):
    g = torch.Generator().manual_seed(N + M + dim + k)
    C, T = 10, 0.1
    mem = F.normalize(torch.randn((M, dim), generator=g), dim=1)
    q = _unit_rows(N, dim, k)
    labels = torch.randint(0, C, (M,), generator=g)
    (sims, idx, preds), counts = TS.launched_kernels(K.bank_topk, q.to(DEV), mem.to(DEV), k, labels.to(DEV), C, T)
    assert kernel == _score_name(k, dim)
    _ran(counts, kernel, "bank_merge_vote_kernel")
    r = _check_topk(q, mem, labels, k, C, T, sims, idx, preds)
    print("RATIO bank_topk N=%d M=%d dim=%d k=%d %.3f" % (N, M, dim, k, r))
    again = K.bank_topk(q.to(DEV), mem.to(DEV), k, labels.to(DEV), C, T)
    assert torch.equal(sims, again[0]) and torch.equal(idx, again[1]) and torch.equal(preds, again[2])


def test_bank_topk_k400_configuration():
    """The trainer's kinetics_k400 kNN memory: 239,975 rows, dim 128, k = 200, 400 classes, T = 0.1; N = 64."""
    g = torch.Generator().manual_seed(400)
    M, dim, k, C, T = 239975, 128, 200, 400, 0.1
    mem = F.normalize(torch.randn((M, dim), generator=g), dim=1)
    q = _unit_rows(64, dim, 401)
    labels = torch.randint(0, C, (M,), generator=g)
    knn = KnnMemory(M, dim, downstream_classes=C, temperature=T, knn_k=k, device=DEV)
    knn.memory.copy_(mem.to(DEV))
    knn.train_labels = labels.to(DEV)
    preds, counts = TS.launched_kernels(knn.eval_knn, q.to(DEV))
    _ran(counts, "bank_score_kernel<topk,32,vec4>", "bank_merge_vote_kernel")
    sims, idx, p2 = K.bank_topk(q.to(DEV), mem.to(DEV), k, labels.to(DEV), C, T)
    assert torch.equal(preds, p2)
    r = _check_topk(q, mem, labels, k, C, T, sims, idx, preds)
    print("RATIO bank_topk k400 %.3f" % r)


def test_bank_topk_ties():
    """Duplicate bank rows, with the same and with different labels: equal similarities by ascending index."""
    dim, M = 64, 3000
    g = torch.Generator().manual_seed(9)
    mem = F.normalize(torch.randn((M, dim), generator=g), dim=1) * 0.1
    q = _unit_rows(2, dim, 10)
    for r in (10, 500, 999, 2999, 1700):
        mem[r] = q[0]
    mem[1200] = q[1]
    mem[40] = q[1]
    labels = torch.randint(0, 5, (M,), generator=g)
    labels[500] = labels[10]
    labels[999] = (labels[10] + 1) % 5
    for k in (1, 3, 5, 300):
        (sims, idx, preds), counts = TS.launched_kernels(K.bank_topk, q.to(DEV), mem.to(DEV), k, labels.to(DEV), 5,
                                                         0.1)
        _ran(counts, _score_name(k, dim))
        assert idx[0, :min(k, 5)].tolist() == [10, 500, 999, 1700, 2999][:k]
        assert idx[1, :min(k, 2)].tolist() == [40, 1200][:k]
        _check_topk(q, mem, labels, k, 5, 0.1, sims, idx, preds)


def test_bank_topk_overflow_row_is_nan():
    """The trainer's stored rows are +-1 (update normalises over a size-1 axis): a unit query's self-similarity is its
    L1 norm, and above 8.87 exp(s / 0.1) overflows; the vote row is +inf in the neighbour's class and NaN elsewhere."""
    dim, M, C, T = 128, 1000, 10, 0.1
    g = torch.Generator().manual_seed(12)
    q = _unit_rows(2, dim, 13)
    assert float(q[0].abs().sum()) > 8.87
    mem = torch.sign(torch.randn((M, dim), generator=g))
    mem[77] = torch.sign(q[0])
    labels = torch.randint(0, C, (M,), generator=g)
    (sims, idx, preds), counts = TS.launched_kernels(K.bank_topk, q.to(DEV), mem.to(DEV), 20, labels.to(DEV), C, T)
    _ran(counts, "bank_score_kernel<topk,32,vec4>", "bank_merge_vote_kernel")
    assert int(idx[0, 0]) == 77
    # the reference's vote on the returned neighbours, in fp32 eager on the CPU
    yd, yi = sims.cpu(), idx.cpu()
    onehot = torch.zeros((2 * 20, C)).scatter_(1, labels[yi].view(-1, 1), 1)
    want = torch.sum(onehot.view(2, -1, C) * yd.clone().div_(T).exp_().view(2, -1, 1), 1)
    assert torch.isinf(want[0, labels[77]]) and int(torch.isnan(want[0]).sum()) == C - 1
    assert torch.allclose(preds.cpu(), want, rtol=1e-5, atol=0, equal_nan=True)


def test_bank_topk_64bit_offsets():
    dim = 2048
    rows = (1 << 31) // dim + 300                          # > 2^31 elements
    need = rows * dim * 4 + (1 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip("needs %.1f GB of free device memory" % (need / 1e9))
    mem = torch.zeros((rows, dim), dtype=torch.float32, device=DEV)
    q = _unit_rows(2, dim, 14)
    mem[rows - 1] = q[0].to(DEV)
    mem[rows - 200] = (0.5 * q[0]).to(DEV)
    mem[3] = (0.25 * q[0]).to(DEV)
    mem[rows - 2] = q[1].to(DEV)
    labels = torch.zeros(rows, dtype=torch.int64, device=DEV)
    (sims, idx, preds), counts = TS.launched_kernels(K.bank_topk, q.to(DEV), mem, 3, labels, 2, 0.1)
    _ran(counts, "bank_score_kernel<topk,32,vec4>")
    assert idx[0].tolist() == [rows - 1, rows - 200, 3]
    assert int(idx[1, 0]) == rows - 2
    del mem
    torch.cuda.empty_cache()


def test_bank_topk_argument_errors():
    q = torch.rand((2, 8), device=DEV)
    mem = torch.rand((100, 8), device=DEV)
    lab = torch.zeros(100, dtype=torch.int64, device=DEV)
    with pytest.raises(RuntimeError):
        K.bank_topk(q, mem, 101, lab, 3, 0.1)
    bad = lab.clone()
    bad[5] = 3
    with pytest.raises(RuntimeError, match="label"):
        K.bank_topk(q, mem, 100, bad, 3, 0.1)


# ---- pv_queue_ce and ContrastiveLoss against float64 ----------------------------------------------------------------
def _ce_tol(dim, L, rows, T, loss):
    return 2 * (2 * (dim + 2) * EPS / T + (L + 8) * EPS + (rows + 4) * EPS * abs(loss) + 4 * EPS / T)


@pytest.mark.parametrize("reduction", ["mean", "none"])
@pytest.mark.parametrize("N,K_,dim,V,skip,kernel", [
    (8, 65536, 128, 2, 0, "bank_score_kernel<lse,32,vec4>"), (32, 65536, 128, 2, 1, "bank_score_kernel<lse,32,vec4>"),
    (5, 1000, 130, 3, 1, "bank_score_kernel<lse,32,scalar>"), (3, 257, 4, 3, -1, "bank_score_kernel<lse,32,vec4>"),
    (1, 1, 2, 1, -1, "bank_score_kernel<lse,32,scalar>")])
def test_queue_ce_vs_f64(reduction, N, K_, dim, V, skip, kernel):
    T = 0.2
    q = _unit_rows(N, dim, 20)
    queue = _unit_rows(K_, dim, 21)
    keys = torch.stack([0.7 * q + 0.3 * _unit_rows(N, dim, 22 + v) for v in range(V)])
    keys = keys / keys.norm(dim=2, keepdim=True)
    blocks = [v for v in range(V) if v != skip]
    rows = []
    for v in blocks:
        lg = torch.cat([(q.double() * keys[v].double()).sum(1, keepdim=True), q.double() @ queue.double().T], 1) / T
        rows.append(torch.logsumexp(lg, 1) - lg[:, 0])
    ref = torch.cat(rows)
    got, counts = TS.launched_kernels(K.queue_ce, q.to(DEV), queue.to(DEV), keys.to(DEV), T, skip, reduction)
    assert kernel.endswith("vec4>") == (dim % 4 == 0)
    _ran(counts, kernel, "queue_ce_rows_kernel")
    if reduction == "mean":
        _ran(counts, "bank_mean_kernel")
        ref = ref.mean()
    tol = _ce_tol(dim, K_ + 1, ref.numel(), T, float(ref.abs().max()))
    err = float((got.cpu().double() - ref).abs().max())
    print("RATIO queue_ce N=%d K=%d dim=%d V=%d %s %.3f" % (N, K_, dim, V, reduction, err / tol))
    assert got.shape == ref.shape and err <= tol
    assert torch.equal(got, K.queue_ce(q.to(DEV), queue.to(DEV), keys.to(DEV), T, skip, reduction))


@pytest.mark.parametrize("reduction", ["mean", "none"])
@pytest.mark.parametrize("R,L", [(1, 1), (7, 300), (64, 4097)])
def test_contrastive_loss_vs_f64(reduction, R, L):
    g = torch.Generator().manual_seed(R * L)
    x = torch.rand((R, L), generator=g) * 2 - 1
    T = 0.1
    lg = x.double() / T
    ref = torch.logsumexp(lg, 1) - lg[:, 0]
    got, counts = TS.launched_kernels(ContrastiveLoss(reduction, T), x.to(DEV))
    _ran(counts, "logits_ce_rows_kernel")
    if reduction == "mean":
        ref = ref.mean()
    tol = _ce_tol(0, L, R, T, float(ref.abs().max()))
    assert got.shape == ref.shape and float((got.cpu().double() - ref).abs().max()) <= tol


def test_knn_memory_update_then_eval():
    """update with the trainer's momentum 1.0 stores sign rows; eval_knn of a stored row's query finds it first."""
    M, dim = 2000, 128
    torch.manual_seed(3)
    knn = KnnMemory(M, dim, momentum=1.0, downstream_classes=10, temperature=0.1, knn_k=5, device=DEV)
    knn.train_labels = torch.randint(0, 10, (M,), device=DEV)
    x = _unit_rows(4, dim, 30).to(DEV) * 1e-3
    ind = torch.tensor([5, 1999, 0, 77], device=DEV)
    before = knn.memory.clone()
    _, counts = TS.launched_kernels(knn.update, x, ind)
    _ran(counts, "bank_update_kernel")
    want = _update_ref(before.cpu(), x.cpu(), ind.cpu(), 1.0)
    assert torch.equal(knn.memory.cpu(), want)
    assert bool((knn.memory[ind].abs() == 1).all())
    probe = torch.sign(x) / math.sqrt(dim)
    preds = knn.eval_knn(probe)
    assert preds.shape == (4, 10)
