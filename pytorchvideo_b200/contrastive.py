"""Host side of the self-supervised objectives (csrc/pv_contrastive.cu): argument checks, output allocation and the
one device-flag read of the memory bank's index check.  Everything is fp32 on the device; nothing here computes with
ATen."""
import ctypes as C

import torch

from . import _lib as L

_DT = {torch.float32: L.PV_F32, torch.float16: L.PV_F16}


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


def _rows(x, what, dtypes=(torch.float32,)):
    if not torch.is_tensor(x) or x.dim() != 2:
        raise RuntimeError("%s must be a 2-D (rows, features) tensor" % what)
    if x.device.type != "cuda":
        raise RuntimeError("pytorchvideo_b200 runs on H100 GPUs only (no CPU path); %s is a %s tensor" % (what, x.device.type))
    if x.dtype not in dtypes:
        raise RuntimeError("%s must be %s, got %s" % (what, " or ".join(str(d) for d in dtypes), x.dtype))
    if x.shape[0] < 1 or x.shape[1] < 1:
        raise RuntimeError("%s is empty" % what)
    if x.stride(1) != 1 or x.stride(0) < x.shape[1]:
        x = x.contiguous()
    return x


def l2_normalize(x, out=None):
    """F.normalize(x, p=2, dim=1) of f16 / f32 rows as fp32 rows (``out``: an fp32 (rows, C) view to write into)."""
    x = _rows(x, "x", (torch.float32, torch.float16))
    R, Cn = x.shape
    if out is None:
        out = torch.empty((R, Cn), dtype=torch.float32, device=x.device)
    elif tuple(out.shape) != (R, Cn) or out.dtype != torch.float32 or out.stride(1) != 1:
        raise RuntimeError("out must be an fp32 (%d, %d) tensor with unit column stride" % (R, Cn))
    L.check(L.load().pv_rows_l2_normalize(x.data_ptr(), _DT[x.dtype], x.stride(0), out.data_ptr(), out.stride(0), R, Cn,
                                          _stream(x.device)), "pv_rows_l2_normalize")
    return out


def contrastive_ce(q, k, temperature, row_offset=0, byol=False):
    """SimCLR (``byol=False``): mean cross entropy of the logits (q @ k.T) / temperature against key row
    ``row_offset + n`` for query row n.  BYOL: -mean_n(q_n . k_n).  fp32 rows; returns a 0-dim fp32 tensor."""
    q, k = _rows(q, "q"), _rows(k, "k")
    N, Cn = q.shape
    M = k.shape[0]
    if k.shape[1] != Cn:
        raise RuntimeError("q has %d features, k %d" % (Cn, k.shape[1]))
    if k.device != q.device:
        raise RuntimeError("q and k are on different devices")
    dev = q.device
    row = torch.empty(N, dtype=torch.float32, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev)
    L.check(L.load().pv_contrastive_ce(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), N, M, Cn, float(temperature),
                                       int(row_offset), 1 if byol else 0, row.data_ptr(), loss.data_ptr(), _stream(dev)),
            "pv_contrastive_ce")
    return loss


def memory_bank_ce(x, memory, idx, temperature):
    """Cross entropy against target 0 of logits[b][j] = (memory[idx[b, j]] . x[b]) / temperature (memory_bank.py:97-103).
    x fp32 (B, dim), memory fp32 (bank_size, dim), idx int64 (B, K1) on the same device.  An index outside the bank
    raises RuntimeError; its row is never read."""
    x = _rows(x, "x")
    memory = _rows(memory, "memory")
    if not memory.is_contiguous():
        memory = memory.contiguous()
    if not torch.is_tensor(idx) or idx.dtype != torch.int64 or idx.dim() != 2 or idx.device != x.device:
        raise RuntimeError("idx must be an int64 (B, K) tensor on the device of x")
    idx = idx.contiguous()
    B, dim = x.shape
    if memory.shape[1] != dim or memory.device != x.device or idx.shape[0] != B:
        raise RuntimeError("shapes do not match: x %s, memory %s, idx %s" % (tuple(x.shape), tuple(memory.shape),
                                                                             tuple(idx.shape)))
    K1 = idx.shape[1]
    dev = x.device
    ws = torch.empty(B * K1 + B + 1, dtype=torch.float32, device=dev)
    flag = torch.empty(1, dtype=torch.int32, device=dev)
    L.check(L.load().pv_memory_bank_ce(x.data_ptr(), x.stride(0), memory.data_ptr(), memory.shape[0], dim, idx.data_ptr(),
                                       B, K1, float(temperature), ws.data_ptr(), ws[B * K1:].data_ptr(),
                                       ws[B * K1 + B:].data_ptr(), flag.data_ptr(), _stream(dev)), "pv_memory_bank_ce")
    if int(flag.item()):
        raise RuntimeError("memory bank index out of range [0, %d)" % memory.shape[0])
    return ws[B * K1 + B]


def soft_target_ce(x, target, normalize_targets=True, eps=torch.finfo(torch.float32).eps, reduction="mean"):
    """Soft-target cross entropy (losses/soft_target_cross_entropy.py:66-81) of (N, C) logits and (N, C) target rows
    (f16 / f32 / int64): (N,) per-sample losses, or their mean as a 0-dim tensor."""
    x = _rows(x, "input", (torch.float32, torch.float16))
    tdt = {torch.float32: L.PV_F32, torch.float16: L.PV_F16, torch.int64: L.PV_I64}
    target = _rows(target, "target", tuple(tdt))
    N, Cn = x.shape
    dev = x.device
    row = torch.empty(N, dtype=torch.float32, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev) if reduction == "mean" else None
    L.check(L.load().pv_soft_target_ce(x.data_ptr(), _DT[x.dtype], x.stride(0), target.data_ptr(), tdt[target.dtype],
                                       target.stride(0), N, Cn, 1 if normalize_targets else 0, float(eps),
                                       1 if loss is not None else 0, row.data_ptr(),
                                       loss.data_ptr() if loss is not None else None, _stream(dev)), "pv_soft_target_ce")
    return row if loss is None else loss


EMA_CHUNK = 4096        # elements per block of pv_ema_update


class EmaUpdate:
    """dst = dst * mmt + src * (1 - mmt) over pairs of fp32 device tensors, one launch (pv_ema_update), in place.  The
    pointer, size and chunk tables are built once: the tensors must keep their storage."""

    def __init__(self, dst, src):
        dst, src = list(dst), list(src)
        if len(dst) != len(src):
            raise RuntimeError("%d momentum tensors for %d tensors" % (len(dst), len(src)))
        for d, s in zip(dst, src):
            if d.shape != s.shape or d.dtype != torch.float32 or s.dtype != torch.float32:
                raise RuntimeError("momentum update needs pairs of fp32 tensors of one shape")
            if d.device.type != "cuda" or s.device != d.device or not d.is_contiguous() or not s.is_contiguous():
                raise RuntimeError("momentum update needs contiguous CUDA tensors on one device")
        self.dst, self.src = dst, src
        self.ptrs = [(d.data_ptr(), s.data_ptr()) for d, s in zip(dst, src)]
        dev = dst[0].device if dst else torch.device("cuda")
        chunks = [(t << 40) | c for t, d in enumerate(dst) for c in range(0, d.numel(), EMA_CHUNK)]
        self.n_chunks = len(chunks)
        self.tab = torch.tensor([p for p, _ in self.ptrs] + [p for _, p in self.ptrs] + [d.numel() for d in dst] + chunks,
                                dtype=torch.int64).to(dev)
        self.n = len(dst)
        self.device = dev

    def __call__(self, mmt):
        if [(d.data_ptr(), s.data_ptr()) for d, s in zip(self.dst, self.src)] != self.ptrs:
            raise RuntimeError("a tensor of the momentum update moved; build a new EmaUpdate")
        if self.n == 0:
            return
        base, n = self.tab.data_ptr(), self.n
        # the reference multiplies by the fp32 scalars mmt and (1.0 - mmt), the latter formed in double precision
        m32 = C.c_float(float(mmt)).value
        omm32 = C.c_float(1.0 - float(mmt)).value
        L.check(L.load().pv_ema_update(base, base + 8 * n, base + 16 * n, base + 24 * n, self.n_chunks, m32, omm32,
                                       _stream(self.device)), "pv_ema_update")


# ---- bank scans (csrc/pv_bank.cu) ------------------------------------------------------------------------------------
KNN_MAX_K = 1024
BANK_MAX_DIM = 2048


def _workspace(op, N, M, k, dev):
    n = C.c_longlong(0)
    L.check(L.load().pv_bank_workspace(op, N, M, k, C.byref(n)), "pv_bank_workspace")
    return torch.empty(max(int(n.value), 16), dtype=torch.uint8, device=dev)


def _bank(memory, dim, what="memory"):
    memory = _rows(memory, what)
    if not memory.is_contiguous():
        memory = memory.contiguous()
    if memory.shape[1] != dim:
        raise RuntimeError("%s has %d features, the queries %d" % (what, memory.shape[1], dim))
    return memory


def bank_topk(q, memory, k, labels, n_classes, temperature):
    """KnnMemory.eval_knn's core (ssl_helper.py:288-311) in two launches (pv_bank_topk): the k largest similarities
    q . m of every fp32 query row against the fp32 bank rows, descending, equal similarities by ascending bank index,
    and the vote preds[n][c] = sum_i onehot(labels[idx_i])[c] * exp(sim_i / temperature).  Returns (sims (N, k) fp32,
    idx (N, k) int64, preds (N, n_classes) fp32).  k <= 1024 and dim <= 2048, else NotImplementedError; k > M raises
    RuntimeError, as torch.topk.  A label outside [0, n_classes) raises RuntimeError."""
    if k > KNN_MAX_K:
        raise NotImplementedError("kNN with k = %d: at most %d neighbours are supported" % (k, KNN_MAX_K))
    if torch.is_tensor(q) and q.dim() == 2 and q.shape[1] > BANK_MAX_DIM:
        raise NotImplementedError("kNN with dim = %d: at most %d features are supported" % (q.shape[1], BANK_MAX_DIM))
    q = _rows(q, "q")
    N, dim = q.shape
    memory = _bank(memory, dim)
    M = memory.shape[0]
    if k < 1 or k > M:
        raise RuntimeError("selected index k = %d out of range for a bank of %d rows" % (k, M))
    if not torch.is_tensor(labels) or labels.dtype != torch.int64 or labels.dim() != 1 or labels.numel() != M:
        raise RuntimeError("labels must be an int64 tensor of the %d bank rows" % M)
    if labels.device != q.device or memory.device != q.device:
        raise RuntimeError("q, memory and labels must be on one device")
    labels = labels.contiguous()
    dev = q.device
    ws = _workspace(0, N, M, k, dev)
    sims = torch.empty((N, k), dtype=torch.float32, device=dev)
    idx = torch.empty((N, k), dtype=torch.int64, device=dev)
    preds = torch.empty((N, n_classes), dtype=torch.float32, device=dev)
    flag = torch.empty(1, dtype=torch.int32, device=dev)
    L.check(L.load().pv_bank_topk(q.data_ptr(), q.stride(0), N, memory.data_ptr(), M, dim, int(k), labels.data_ptr(),
                                  int(n_classes), float(temperature), ws.data_ptr(), ws.numel(), sims.data_ptr(),
                                  idx.data_ptr(), preds.data_ptr(), flag.data_ptr(), _stream(dev)), "pv_bank_topk")
    if int(flag.item()):
        raise RuntimeError("a neighbour's label is outside [0, %d)" % n_classes)
    return sims, idx, preds


def bank_update(memory, x, ind, momentum):
    """KnnMemory.update's write (ssl_helper.py:245-250), in place, one launch (pv_bank_update): memory[ind[n]] =
    v / max(|v|, 1e-12) elementwise with v = x[n] * momentum + memory[ind[n]] * (1 - momentum) in fp32 (the scalars
    rounded to fp32 as torch does), every row blended against the bank as it was before the call; of repeated indices
    the last occurrence wins.  An index outside the bank raises RuntimeError and nothing is written."""
    if not torch.is_tensor(memory) or memory.dim() != 2 or not memory.is_contiguous() or memory.dtype != torch.float32:
        raise RuntimeError("memory must be a contiguous fp32 (rows, dim) tensor")
    x = _rows(x, "x")
    M, dim = memory.shape
    if x.shape[1] != dim or x.device != memory.device:
        raise RuntimeError("x %s does not match the memory %s" % (tuple(x.shape), tuple(memory.shape)))
    if not torch.is_tensor(ind) or ind.dtype != torch.int64 or ind.numel() != x.shape[0] or ind.device != x.device:
        raise RuntimeError("ind must be an int64 tensor of one index per row of x on its device")
    ind = ind.reshape(-1).contiguous()
    dev = x.device
    flag = torch.empty(1, dtype=torch.int32, device=dev)
    m32 = C.c_float(float(momentum)).value
    omm32 = C.c_float(1 - float(momentum)).value
    L.check(L.load().pv_bank_update(x.data_ptr(), x.stride(0), x.shape[0], ind.data_ptr(), memory.data_ptr(), M, dim,
                                    m32, omm32, flag.data_ptr(), _stream(dev)), "pv_bank_update")
    if int(flag.item()):
        raise RuntimeError("memory index out of range [0, %d)" % M)
    return memory


def queue_ce(q, queue, keys, temperature, skip_view=-1, reduction="mean"):
    """MoCo's objective (moco_v2.py:312-323 with ContrastiveLoss): q fp32 (N, dim) query rows, queue fp32 (K, dim),
    keys fp32 (V, N, dim).  For every view v != skip_view (-1: none), in order, row (j, n) has the logits
    [q_n . keys[v, n], q_n . queue_0, ..., q_n . queue_K-1] / temperature and target 0; the ((V - 1) N, 1 + K) logits
    are never stored.  Returns the mean (0-dim) or the (rows,) losses."""
    if reduction not in ("mean", "none"):
        raise NotImplementedError('reduction type "%s" not implemented' % reduction)
    if torch.is_tensor(q) and q.dim() == 2 and q.shape[1] > BANK_MAX_DIM:
        raise NotImplementedError("queue cross entropy with dim = %d: at most %d features" % (q.shape[1], BANK_MAX_DIM))
    q = _rows(q, "q")
    N, dim = q.shape
    queue = _bank(queue, dim, "queue")
    if not torch.is_tensor(keys) or keys.dim() != 3 or tuple(keys.shape[1:]) != (N, dim) or \
            keys.dtype != torch.float32 or keys.device != q.device:
        raise RuntimeError("keys must be an fp32 (V, %d, %d) tensor on the device of q" % (N, dim))
    keys = keys.contiguous()
    V = keys.shape[0]
    if not -1 <= skip_view < V or V - (skip_view >= 0) < 1:
        raise RuntimeError("no positive key block: V = %d, skip_view = %d" % (V, skip_view))
    dev = q.device
    rows = (V - (skip_view >= 0)) * N
    ws = _workspace(1, N, queue.shape[0], 1, dev)
    row = torch.empty(rows, dtype=torch.float32, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev) if reduction == "mean" else None
    L.check(L.load().pv_queue_ce(q.data_ptr(), q.stride(0), N, dim, queue.data_ptr(), queue.shape[0], keys.data_ptr(),
                                 dim, V, int(skip_view), None, 0, 0, float(temperature), ws.data_ptr(), ws.numel(),
                                 1 if loss is not None else 0, row.data_ptr(),
                                 loss.data_ptr() if loss is not None else None, _stream(dev)), "pv_queue_ce")
    return row if loss is None else loss


def logits_ce(logits, temperature, reduction="mean"):
    """ContrastiveLoss(inputs) (losses.py:125-134) on materialised fp32 (R, L) logits: cross entropy of
    logits / temperature against target 0 (pv_queue_ce).  The mean (0-dim) or the (R,) losses."""
    if reduction not in ("mean", "none"):
        raise NotImplementedError('reduction type "%s" not implemented' % reduction)
    x = _rows(logits, "inputs")
    R, Ln = x.shape
    dev = x.device
    row = torch.empty(R, dtype=torch.float32, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev) if reduction == "mean" else None
    L.check(L.load().pv_queue_ce(None, 0, R, 0, None, 0, None, 0, 0, -1, x.data_ptr(), x.stride(0), Ln,
                                 float(temperature), None, 0, 1 if loss is not None else 0, row.data_ptr(),
                                 loss.data_ptr() if loss is not None else None, _stream(dev)), "pv_queue_ce")
    return row if loss is None else loss
